// ORACLE (test infrastructure, NOT product code).  Parity unpinned (see so3.hpp).
// C entry points of the CPU oracle (liboracle.so).  They mirror include/ctvio.h
// one-to-one with the prefix `ctvo_` so that tests drive the CUDA engine and
// the oracle from identical inputs; the struct layouts are taken from the
// product's PUBLIC header (the dependency points from the checker to the
// product's interface, never the other way).
#include <cstring>
#include <string>

#include "../include/ctvio.h"
#include "engine.hpp"
#include "triangulate.hpp"

using namespace ctvio_oracle;

namespace {
struct OracleEngine {
  Window w;
  bool have_cfg = false;
  std::vector<double> sq, sp, sbias, srho;  // snapshot
  double sld = 0;
};
thread_local std::string g_err;
int fail(int code, const char* msg) {
  g_err = msg;
  return code;
}
OracleEngine* E(void* h) { return reinterpret_cast<OracleEngine*>(h); }
}  // namespace

extern "C" {

const char* ctvo_last_error(void) { return g_err.c_str(); }
int ctvo_abi_version(void) { return CTVIO_ABI_VERSION; }

int ctvo_create(const ctvio_config* cfg, void** out) {
  if (!cfg || !out) return fail(CTVIO_ERR_INVALID, "null argument");
  if (cfg->dt_ns <= 0) return fail(CTVIO_ERR_INVALID, "dt_ns must be positive");
  auto* e = new OracleEngine();
  e->w.grid.set(cfg->t0_ns, cfg->dt_ns, 0);
  e->w.cal.S_CtoI = Quat::fromPtr(cfg->q_CtoI);
  e->w.cal.p_CinI = Vec3(cfg->p_CinI[0], cfg->p_CinI[1], cfg->p_CinI[2]);
  e->w.cal.sqrt_info = cfg->image_weight;
  e->w.cal.gravity = Vec3(cfg->gravity[0], cfg->gravity[1], cfg->gravity[2]);
  for (int k = 0; k < 6; ++k) e->w.cal.imu_info[k] = cfg->imu_info[k];
  e->w.opt.rs_padding_ns = cfg->rs_padding_ns;
  e->w.opt.cauchy_solve = cfg->cauchy_solve;
  e->w.opt.cauchy_marg = cfg->cauchy_marg;
  e->have_cfg = true;
  *out = e;
  return CTVIO_OK;
}
int ctvo_destroy(void* h) {
  delete E(h);
  return CTVIO_OK;
}
int ctvo_set_options(void* h, const ctvio_options* o) {
  if (!h || !o) return fail(CTVIO_ERR_INVALID, "null argument");
  Options& t = E(h)->w.opt;
  t.fixed_knot_index = o->fixed_knot_index;
  t.lock_traj = o->lock_traj != 0;
  t.lock_wb = o->lock_wb != 0;
  t.lock_ab = o->lock_ab != 0;
  t.fix_ld = o->fix_ld != 0;
  t.is_marg_state = o->is_marg_state != 0;
  t.ctrl_to_be_opt_now = o->ctrl_to_be_opt_now;
  t.ctrl_to_be_opt_later = o->ctrl_to_be_opt_later;
  t.ld_lower = o->ld_lower;
  t.ld_upper = o->ld_upper;
  return CTVIO_OK;
}
int ctvo_set_num_threads(void* h, int32_t n) {
  E(h)->w.opt.num_threads = n;
  return CTVIO_OK;
}
int ctvo_set_knots(void* h, int32_t n, const double* q, const double* p) {
  Window& w = E(h)->w;
  w.q.assign(q, q + 4 * size_t(n));
  w.p.assign(p, p + 3 * size_t(n));
  w.grid.set(w.grid.t0_ns, w.grid.dt_ns, n);
  return CTVIO_OK;
}
int ctvo_set_biases(void* h, int32_t n, const double* b) {
  E(h)->w.bias.assign(b, b + 6 * size_t(n));
  return CTVIO_OK;
}
int ctvo_set_inv_depths(void* h, int32_t n, const double* r) {
  E(h)->w.rho.assign(r, r + size_t(n));
  return CTVIO_OK;
}
int ctvo_set_time_origin(void* h, int64_t t0_ns) {
  Window& w = E(h)->w;
  if ((t0_ns - w.grid.t0_ns) % w.grid.dt_ns != 0) return fail(CTVIO_ERR_INVALID, "time origin off the knot grid");
  w.grid.set(t0_ns, w.grid.dt_ns, w.grid.n_knots);
  return CTVIO_OK;
}
int ctvo_set_line_delay(void* h, double ld) {
  E(h)->w.ld = ld;
  return CTVIO_OK;
}
int ctvo_get_knots(void* h, double* q, double* p) {
  Window& w = E(h)->w;
  if (q) std::memcpy(q, w.q.data(), w.q.size() * sizeof(double));
  if (p) std::memcpy(p, w.p.data(), w.p.size() * sizeof(double));
  return CTVIO_OK;
}
int ctvo_get_biases(void* h, double* b) {
  Window& w = E(h)->w;
  std::memcpy(b, w.bias.data(), w.bias.size() * sizeof(double));
  return CTVIO_OK;
}
int ctvo_get_inv_depths(void* h, double* r) {
  Window& w = E(h)->w;
  std::memcpy(r, w.rho.data(), w.rho.size() * sizeof(double));
  return CTVIO_OK;
}
int ctvo_get_line_delay(void* h, double* ld) {
  *ld = E(h)->w.ld;
  return CTVIO_OK;
}
int ctvo_clear_factors(void* h) {
  Window& w = E(h)->w;
  w.img.clear();
  w.imu.clear();
  w.biasf.clear();
  return CTVIO_OK;
}
int ctvo_add_image_features(void* h, int32_t n, const int64_t* ti, const int32_t* rowi, const double* pi,
                            const int64_t* tj, const int32_t* rowj, const double* pj, const int32_t* lm,
                            const int32_t* marg) {
  Window& w = E(h)->w;
  for (int k = 0; k < n; ++k) {
    ImageObs o;
    o.ti = ti[k]; o.tj = tj[k]; o.rowi = rowi[k]; o.rowj = rowj[k];
    o.pi[0] = pi[2 * k]; o.pi[1] = pi[2 * k + 1];
    o.pj[0] = pj[2 * k]; o.pj[1] = pj[2 * k + 1];
    o.lm = lm[k];
    o.marg = marg ? marg[k] : 0;
    if (o.lm < 0 || o.lm >= w.nL()) return fail(CTVIO_ERR_INVALID, "landmark index out of range");
    w.img.push_back(o);
  }
  return CTVIO_OK;
}
int ctvo_add_imu_measurements(void* h, int32_t n, const int64_t* t, const double* gyro, const double* accel,
                              const int32_t* node, const int32_t* marg) {
  Window& w = E(h)->w;
  for (int k = 0; k < n; ++k) {
    ImuObs o;
    o.t = t[k];
    for (int c = 0; c < 3; ++c) {
      o.gyro[c] = gyro[3 * k + c];
      o.accel[c] = accel[3 * k + c];
    }
    o.bias_idx = node[k];
    o.marg = marg ? marg[k] : 0;
    if (o.bias_idx < 0 || o.bias_idx >= w.nB()) return fail(CTVIO_ERR_INVALID, "bias node out of range");
    w.imu.push_back(o);
  }
  return CTVIO_OK;
}
int ctvo_add_bias_factors(void* h, int32_t n, const int32_t* ni, const int32_t* nj, const double* si,
                          const int32_t* marg) {
  Window& w = E(h)->w;
  for (int k = 0; k < n; ++k) {
    BiasObs o;
    o.i = ni[k]; o.j = nj[k];
    for (int c = 0; c < 6; ++c) o.sqrt_info[c] = si[6 * k + c];
    o.marg = marg ? marg[k] : 0;
    w.biasf.push_back(o);
  }
  return CTVIO_OK;
}
int ctvo_set_prior(void* h, int32_t n, const double* J, const double* r, int32_t nb, const int32_t* type,
                   const int32_t* index, const int32_t* col, const double* x0) {
  Prior& p = E(h)->w.prior;
  p = Prior();
  if (n <= 0) return CTVIO_OK;
  p.n = n;
  p.J.assign(J, J + size_t(n) * n);
  p.r.assign(r, r + n);
  for (int b = 0; b < nb; ++b) {
    PriorBlock pb;
    pb.type = type[b]; pb.index = index[b]; pb.col = col[b];
    for (int d = 0; d < 4; ++d) pb.x0[d] = x0[4 * b + d];
    p.blocks.push_back(pb);
  }
  return CTVIO_OK;
}
int ctvo_solve(void* h, int32_t max_iterations, ctvio_summary* s) {
  Window& w = E(h)->w;
  if (w.nK() < kN) return fail(CTVIO_ERR_STATE, "need at least 4 knots");
  Summary r = w.solve(max_iterations);
  if (s) {
    std::memset(s, 0, sizeof(*s));
    s->iterations = r.iterations;
    s->num_successful_steps = r.num_successful_steps;
    s->num_unsuccessful_steps = r.num_unsuccessful_steps;
    s->termination = r.termination;
    s->num_cost_evals = r.num_cost_evals;
    s->num_jacobian_evals = r.num_jacobian_evals;
    s->num_linear_solves = r.num_linear_solves;
    s->num_line_search_steps = r.num_line_search_steps;
    s->initial_cost = r.initial_cost;
    s->final_cost = r.final_cost;
    s->final_radius = r.final_radius;
    s->device_ms = r.t_total_s * 1e3;  // host wall-clock of the CPU solve
    s->kernel_launches = 0;
  }
  return CTVIO_OK;
}
// breakdown of the last solve is not kept; a dedicated timing entry point for bench's cpu_baseline
int ctvo_solve_timed(void* h, int32_t max_iterations, double* out4) {
  Summary r = E(h)->w.solve(max_iterations);
  out4[0] = r.t_total_s; out4[1] = r.t_eval_s; out4[2] = r.t_schur_s; out4[3] = r.t_solve_s;
  return r.iterations;
}
int ctvo_gauge_realign(void* h, int32_t min_idx, const double* R0, const double* t0) {
  E(h)->w.gauge_realign(min_idx, R0, t0);
  return CTVIO_OK;
}
int ctvo_marginalize(void* h, int32_t* n_out, int32_t* nb_out) {
  Window& w = E(h)->w;
  const bool ok = w.marginalize();
  *n_out = ok ? w.new_prior.n : 0;
  *nb_out = ok ? int(w.new_prior.blocks.size()) : 0;
  return CTVIO_OK;
}
int ctvo_get_prior(void* h, double* J, double* r, int32_t* type, int32_t* index, int32_t* col, double* x0) {
  const Prior& p = E(h)->w.new_prior;
  if (J) std::memcpy(J, p.J.data(), p.J.size() * sizeof(double));
  if (r) std::memcpy(r, p.r.data(), p.r.size() * sizeof(double));
  for (size_t b = 0; b < p.blocks.size(); ++b) {
    if (type) type[b] = p.blocks[b].type;
    if (index) index[b] = p.blocks[b].index;
    if (col) col[b] = p.blocks[b].col;
    if (x0) for (int d = 0; d < 4; ++d) x0[4 * b + d] = p.blocks[b].x0[d];
  }
  return CTVIO_OK;
}
int ctvo_adopt_prior(void* h) {
  Window& w = E(h)->w;
  w.prior = w.new_prior;
  return CTVIO_OK;
}
int ctvo_save_state(void* h) {
  OracleEngine* e = E(h);
  e->sq = e->w.q; e->sp = e->w.p; e->sbias = e->w.bias; e->srho = e->w.rho; e->sld = e->w.ld;
  return CTVIO_OK;
}
int ctvo_restore_state(void* h) {
  OracleEngine* e = E(h);
  e->w.q = e->sq; e->w.p = e->sp; e->w.bias = e->sbias; e->w.rho = e->srho; e->w.ld = e->sld;
  return CTVIO_OK;
}

int ctvo_eval_image_factors(void* h, int32_t want_jac, double cauchy, double* r, int32_t* s, double* J,
                            double* cost) {
  Window& w = E(h)->w;
  double c = 0;
  for (size_t n = 0; n < w.img.size(); ++n) {
    ImageEval e;
    std::memset(&e, 0, sizeof(e));
    EvaluateImage(w.grid, w.cal, w.q.data(), w.p.data(), w.rho[w.img[n].lm], w.ld, w.img[n], want_jac != 0, e);
    if (!e.ok) return fail(CTVIO_ERR_TIME_RANGE, "image factor time outside the spline");
    if (cauchy > 0) c += ApplyLossImage(cauchy, e, want_jac != 0);
    else c += 0.5 * (e.r[0] * e.r[0] + e.r[1] * e.r[1]);
    if (r) { r[2 * n] = e.r[0]; r[2 * n + 1] = e.r[1]; }
    if (s) { s[2 * n] = int32_t(e.s[0]); s[2 * n + 1] = int32_t(e.s[1]); }
    if (J && want_jac) {
      double* o = J + 100 * n;
      for (int side = 0; side < 2; ++side)
        for (int k = 0; k < 4; ++k) {
          for (int c2 = 0; c2 < 6; ++c2) o[(side * 4 + k) * 12 + c2] = e.Jrot[side][k][c2];
          for (int c2 = 0; c2 < 6; ++c2) o[(side * 4 + k) * 12 + 6 + c2] = e.Jpos[side][k][c2];
        }
      o[96] = e.Jrho[0]; o[97] = e.Jrho[1]; o[98] = e.Jld[0]; o[99] = e.Jld[1];
    }
  }
  if (cost) *cost = c;
  return CTVIO_OK;
}
int ctvo_eval_imu_factors(void* h, int32_t want_jac, double* r, int32_t* s, double* J, double* cost) {
  Window& w = E(h)->w;
  double c = 0;
  for (size_t n = 0; n < w.imu.size(); ++n) {
    const ImuObs& o = w.imu[n];
    ImuEval e;
    std::memset(&e, 0, sizeof(e));
    EvaluateImu(w.grid, w.cal, w.q.data(), w.p.data(), &w.bias[6 * o.bias_idx], &w.bias[6 * o.bias_idx + 3], o,
                want_jac != 0, e);
    if (!e.ok) return fail(CTVIO_ERR_TIME_RANGE, "imu factor time outside the spline");
    for (int k = 0; k < 6; ++k) c += 0.5 * e.r[k] * e.r[k];
    if (r) for (int k = 0; k < 6; ++k) r[6 * n + k] = e.r[k];
    if (s) s[n] = int32_t(e.s);
    if (J && want_jac) {
      double* out = J + 156 * n;
      for (int k = 0; k < 4; ++k) {
        for (int c2 = 0; c2 < 18; ++c2) out[k * 36 + c2] = e.Jrot[k][c2];
        for (int c2 = 0; c2 < 18; ++c2) out[k * 36 + 18 + c2] = e.Jpos[k][c2];
      }
      for (int k = 0; k < 3; ++k) {
        out[144 + k] = e.Jbg[k];
        out[147 + k] = 0.0;
        out[150 + k] = 0.0;
        out[153 + k] = e.Jba[3 + k];
      }
    }
  }
  if (cost) *cost = c;
  return CTVIO_OK;
}
int ctvo_eval_cost(void* h, double* cost) {
  Window& w = E(h)->w;
  NormalEq ne;
  w.buildStructure(&ne);
  *cost = w.assemble(Window::kCost, &ne);
  return CTVIO_OK;
}
int ctvo_normal_equations(void* h, double* Hcc, double* gc, double* hl, double* gl, double* cost) {
  Window& w = E(h)->w;
  NormalEq ne;
  w.buildStructure(&ne);
  const double c = w.assemble(Window::kFull, &ne);
  const int np = ne.np;
  if (Hcc)
    for (int i = 0; i < np; ++i)
      for (int j = i; j < np; ++j) Hcc[size_t(i) * np + j] = Hcc[size_t(j) * np + i] = ne.Hcc[size_t(i) * np + j];
  if (gc) std::memcpy(gc, ne.gc.data(), np * sizeof(double));
  if (hl) std::memcpy(hl, ne.hl.data(), ne.nL * sizeof(double));
  if (gl) std::memcpy(gl, ne.gl.data(), ne.nL * sizeof(double));
  if (cost) *cost = c;
  return CTVIO_OK;
}
// Dense per-landmark coupling rows W (nL x np) for small parity cases.
int ctvo_landmark_coupling(void* h, double* Wdense) {
  Window& w = E(h)->w;
  NormalEq ne;
  w.buildStructure(&ne);
  w.assemble(Window::kFull, &ne);
  const int np = ne.np;
  std::memset(Wdense, 0, sizeof(double) * size_t(ne.nL) * np);
  for (int l = 0; l < ne.nL; ++l) {
    for (int a = ne.lo[l]; a < ne.hi[l]; ++a) Wdense[size_t(l) * np + a] = ne.W[ne.woff[l] + (a - ne.lo[l])];
    Wdense[size_t(l) * np + w.idxLd()] = ne.wld[l];
  }
  return CTVIO_OK;
}

int ctvo_query_trajectory(void* h, int32_t n, const int64_t* t, double* q, double* p, double* omega, double* vel,
                          double* acc) {
  Window& w = E(h)->w;
  for (int k = 0; k < n; ++k) {
    int64_t s; double u;
    if (!w.grid.computeTIndexNs(t[k], s, u)) return fail(CTVIO_ERR_TIME_RANGE, "query time outside the spline");
    if (q) EvaluateRp(w.grid, w.q.data(), t[k], nullptr).toPtr(q + 4 * k);
    if (p) { Vec3 v = RdEvaluate<0>(w.grid, w.p.data(), t[k], nullptr); p[3 * k] = v.x; p[3 * k + 1] = v.y; p[3 * k + 2] = v.z; }
    if (omega) { Vec3 v = VelocityBody(w.grid, w.q.data(), t[k], nullptr); omega[3 * k] = v.x; omega[3 * k + 1] = v.y; omega[3 * k + 2] = v.z; }
    if (vel) { Vec3 v = RdEvaluate<1>(w.grid, w.p.data(), t[k], nullptr); vel[3 * k] = v.x; vel[3 * k + 1] = v.y; vel[3 * k + 2] = v.z; }
    if (acc) { Vec3 v = RdEvaluate<2>(w.grid, w.p.data(), t[k], nullptr); acc[3 * k] = v.x; acc[3 * k + 1] = v.y; acc[3 * k + 2] = v.z; }
  }
  return CTVIO_OK;
}

int ctvo_triangulate(void*, int32_t n_frames, const double* Rs, const double* Ps, const double* ric, const double* tic,
                     int32_t nl, const int32_t* start_frame, const int32_t* obs_offset, const double* obs_point,
                     int32_t window_size, double init_depth, double* depth) {
  triangulate(n_frames, Rs, Ps, ric, tic, nl, start_frame, obs_offset, obs_point, window_size, init_depth, depth);
  return CTVIO_OK;
}

int ctvo_selfcheck_solver(void*, int32_t, int32_t* mm, double* res) {
  if (mm) *mm = 0;
  if (res) *res = 0.0;
  return 0;
}
int ctvo_measure_fp64_tflops(void*, double* v) {
  *v = 0.0;
  return CTVIO_OK;
}
int ctvo_measure_fp64_tensor_tflops(void*, double* v) {
  *v = 0.0;
  return CTVIO_OK;
}
int ctvo_profile_kernels(void*, int32_t, int32_t, double* out) {
  for (int k = 0; k < 8; ++k) out[k] = 0.0;  // not meaningful for the CPU oracle
  return CTVIO_OK;
}

// ---- oracle-only probes for the self-validation tests ------------------------------------------
// kind: 0 EvaluateRp, 1 EvaluateRTp, 2 VelocityBody, 3 EvaluateRotation.  out_val: quat(4) or vec3;
// out_J: 4 x 9 row-major blocks, start index returned.
int ctvo_probe_so3_view(void* h, int32_t kind, int64_t t, double* out_val, double* out_J) {
  Window& w = E(h)->w;
  So3Jacobian J;
  for (auto& m : J.d_val_d_knot) m = Mat3::Zero();
  if (kind == 0) EvaluateRp(w.grid, w.q.data(), t, &J).toPtr(out_val);
  else if (kind == 1) EvaluateRTp(w.grid, w.q.data(), t, &J).toPtr(out_val);
  else if (kind == 3) EvaluateRotation(w.grid, w.q.data(), t, &J).toPtr(out_val);
  else { Vec3 v = VelocityBody(w.grid, w.q.data(), t, &J); out_val[0] = v.x; out_val[1] = v.y; out_val[2] = v.z; }
  if (out_J) for (int k = 0; k < 4; ++k) std::memcpy(out_J + 9 * k, J.d_val_d_knot[k].m, 9 * sizeof(double));
  return int(J.start_idx);
}
// plain-spline evaluators (independent second implementation): q(4), omega(3), alpha(3)
int ctvo_probe_plain_so3(void* h, int64_t t, double* q, double* omega, double* alpha) {
  Window& w = E(h)->w;
  PlainSo3Evaluate(w.grid, w.q.data(), t).toPtr(q);
  Vec3 v = PlainSo3VelocityBody(w.grid, w.q.data(), t);
  omega[0] = v.x; omega[1] = v.y; omega[2] = v.z;
  v = PlainSo3AccelerationBody(w.grid, w.q.data(), t);
  alpha[0] = v.x; alpha[1] = v.y; alpha[2] = v.z;
  return 0;
}
// SplitSpineView::Evaluate: gyro(3), accel(3), J_rot_w (4x9), J_rot_a (4x9), J_pos (4)
int ctvo_probe_split(void* h, int64_t t, double* gyro, double* accel, double* Jw, double* Ja, double* Jp) {
  Window& w = E(h)->w;
  So3Jacobian jw, ja;
  RdJacobian jp;
  SplineIMUData d = SplitEvaluate(w.grid, w.q.data(), w.p.data(), t, w.cal.gravity, &jw, &ja, &jp);
  for (int k = 0; k < 3; ++k) { gyro[k] = d.gyro[k]; accel[k] = d.accel[k]; }
  for (int k = 0; k < 4; ++k) {
    std::memcpy(Jw + 9 * k, jw.d_val_d_knot[k].m, 9 * sizeof(double));
    std::memcpy(Ja + 9 * k, ja.d_val_d_knot[k].m, 9 * sizeof(double));
    Jp[k] = jp.d_val_d_knot[k];
  }
  return int(d.start_idx);
}
// SO(3) leaf math probes: exp (in 3 -> out 4), log (in 4 -> out 3), Jr, JrInv (in 3 -> out 9)
int ctvo_probe_so3(int32_t kind, const double* in, double* out) {
  if (kind == 0) so3_exp(Vec3(in[0], in[1], in[2])).toPtr(out);
  else if (kind == 1) { Vec3 v = so3_log(Quat::fromPtr(in)); out[0] = v.x; out[1] = v.y; out[2] = v.z; }
  else if (kind == 2) { Mat3 m = rightJacobianSO3(Vec3(in[0], in[1], in[2])); std::memcpy(out, m.m, sizeof(m.m)); }
  else if (kind == 3) { Mat3 m = rightJacobianInvSO3(Vec3(in[0], in[1], in[2])); std::memcpy(out, m.m, sizeof(m.m)); }
  else if (kind == 4) { Quat q = so3_mul(Quat::fromPtr(in), Quat::fromPtr(in + 4)); q.toPtr(out); }
  else if (kind == 5) { Vec3 v = so3_rotate(Quat::fromPtr(in), Vec3(in[4], in[5], in[6])); out[0] = v.x; out[1] = v.y; out[2] = v.z; }
  else if (kind == 6) { Mat3 m = so3_matrix(Quat::fromPtr(in)); std::memcpy(out, m.m, sizeof(m.m)); }
  return 0;
}

}  // extern "C"
