// The prior and the marginalization (K7, kernels in marginalize.cu) on the host: the active prior's preparation for the
// factor kernels, the C-ABI that sets, reads, adopts and enables it, and ctvio_marginalize in its stages (block
// discovery and positions, row assembly, the Schur complement, the new prior).  The block rules are param_blocks.h.
#include <algorithm>

#include "engine_state.h"

namespace ctvio::host {

// prepare()'s last stage: the active prior's tables and J'J on the device, and its columns' camera dims (col2g, -1 for
// the constant ones)
int prepare_prior(ctvio_engine* e) {
  const ProblemDims d = e->dims();
  const ctvio::PriorHost& pr = e->prior;
  e->prior_dirty = false;
  if (pr.n <= 0) return CTVIO_OK;
  cudaStream_t st = e->stream;
  std::vector<int32_t> col2g(pr.n, -1);
  for (size_t b = 0; b < pr.type.size(); ++b) {
    const int g = ctvio::block_base(pr.type[b], pr.index[b], d.nK, d.nB);
    if (pr.type[b] == CTVIO_BLK_RHO) return fail(CTVIO_ERR_INVALID, "inverse-depth blocks cannot be part of a prior");
    if (g < 0) return fail(CTVIO_ERR_INVALID, "prior block index out of range");
    for (int c = 0; c < ctvio::block_dim(pr.type[b]); ++c)
      if (!e->h_cmask[g + c]) col2g[pr.col[b] + c] = g + c;
  }
  if (!e->prior_on_device) {
    CUDA_OK(e->d_prior_J.upload(pr.J, st));
    CUDA_OK(e->d_prior_r.upload(pr.r, st));
    CUDA_OK(e->d_prior_x0.upload(pr.x0, st));
  }
  CUDA_OK(e->d_prior_type.upload(pr.type, st));
  CUDA_OK(e->d_prior_index.upload(pr.index, st));
  CUDA_OK(e->d_prior_col.upload(pr.col, st));
  CUDA_OK(e->d_prior_col2g.upload(col2g, st));
  CUDA_OK(e->d_prior_JtJ.reserve(size_t(pr.n) * pr.n));
  CUDA_OK(e->d_prior_dx.reserve(pr.n));
  CUDA_OK(e->d_prior_res.reserve(pr.n));
  CUDA_OK(cudaMemsetAsync(e->d_prior_dx.p, 0, size_t(pr.n) * sizeof(double), st));
  e->launches += ctvio::launch_gram(e->d_prior_J.p, pr.n, pr.n, e->d_prior_JtJ.p, st);
  return CTVIO_OK;
}

// make sure the host copy of the freshly marginalized prior exists (ctvio_get_prior; the device-to-device hand-over of
// ctvio_adopt_prior never needs it)
int fetch_new_prior(ctvio_engine* e) {
  ctvio::PriorHost& np_ = e->new_prior;
  if (e->new_prior_on_host || np_.n <= 0) return CTVIO_OK;
  np_.J.resize(size_t(np_.n) * np_.n);
  np_.r.resize(np_.n);
  np_.x0.resize(4 * np_.type.size());
  CUDA_OK(cudaMemcpyAsync(np_.J.data(), e->mws.J.p, np_.J.size() * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(cudaMemcpyAsync(np_.r.data(), e->mws.r.p, np_.r.size() * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(cudaMemcpyAsync(np_.x0.data(), e->d_newprior_x0.p, np_.x0.size() * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(stream_sync(e->stream));
  e->d2h_bytes += (np_.J.size() + np_.r.size() + np_.x0.size()) * sizeof(double);
  e->new_prior_on_host = true;
  return CTVIO_OK;
}

PriorPtrs prior_ptrs(ctvio_engine* e) {
  PriorPtrs p;
  std::memset(&p, 0, sizeof(p));
  p.n = e->prior_enabled ? e->prior.n : 0;
  if (p.n <= 0) return p;
  p.n_blocks = int(e->prior.type.size());
  p.J = e->d_prior_J.p; p.r = e->d_prior_r.p; p.JtJ = e->d_prior_JtJ.p;
  p.type = e->d_prior_type.p; p.index = e->d_prior_index.p; p.col = e->d_prior_col.p;
  p.x0 = e->d_prior_x0.p; p.col2g = e->d_prior_col2g.p;
  p.dx = e->d_prior_dx.p; p.res = e->d_prior_res.p;
  return p;
}

// ctvio_adopt_prior.  keep_new_prior: the marginalization's buffers are copied device-to-device instead of handed over,
// so that ctvio_get_prior still returns the prior just produced (the odometry cycle)
int adopt_prior_body(ctvio_engine* e, bool keep_new_prior) {
  // only the block bookkeeping (a few dozen ints) lives on the host
  e->prior.n = e->new_prior.n;
  e->prior.type = e->new_prior.type; e->prior.index = e->new_prior.index; e->prior.col = e->new_prior.col;
  e->prior.J.clear(); e->prior.r.clear(); e->prior.x0.clear();
  if (keep_new_prior) {
    const size_t n = size_t(e->new_prior.n), nb = e->new_prior.type.size();
    CUDA_OK(e->d_prior_J.reserve(n * n)); CUDA_OK(e->d_prior_r.reserve(n)); CUDA_OK(e->d_prior_x0.reserve(4 * nb));
    CUDA_OK(cudaMemcpyAsync(e->d_prior_J.p, e->mws.J.p, n * n * sizeof(double), cudaMemcpyDeviceToDevice, e->stream));
    CUDA_OK(cudaMemcpyAsync(e->d_prior_r.p, e->mws.r.p, n * sizeof(double), cudaMemcpyDeviceToDevice, e->stream));
    CUDA_OK(cudaMemcpyAsync(e->d_prior_x0.p, e->d_newprior_x0.p, 4 * nb * sizeof(double), cudaMemcpyDeviceToDevice, e->stream));
  } else {
    // the buffers of the marginalization workspace BECOME the active prior (pointer swap)
    swap(e->d_prior_J, e->mws.J); swap(e->d_prior_r, e->mws.r); swap(e->d_prior_x0, e->d_newprior_x0);
    e->new_prior = ctvio::PriorHost();  // its device buffers are gone
  }
  e->prior_on_device = true;
  e->prior_dirty = true;
  e->masks_dirty = true;
  return CTVIO_OK;
}

namespace {

// ---- ctvio_marginalize's stages ----

// a parameter block the recorded factors or the old prior touch, stored at its first camera dim
struct MargBlock {
  int type = -1, index = 0;  // type -1: no block starts at this dim
  bool dropped = false;
  int pos = -1;              // first position in the [dropped | dropped inverse depths | kept] ordering
};

// what block discovery finds, for the later stages
struct MargPlan {
  std::vector<MargBlock> blocks;  // [np]: in camera-dim order, which is the block order
  bool use_prior = false;         // the old prior has a dropped block and is recorded
  int n_marg = 0, n_rho = 0;      // recorded image factors, their dropped inverse depths
  int m = 0, n = 0, P = 0;        // dropped dims (inverse depths included), kept dims, both
  std::vector<int32_t> marg_img, pos_lm;  // host-built image factors only
  std::vector<int32_t> marg_imu, pos_cam, prior_pos;
  std::vector<int2> bij;
  std::vector<double> bs;
  std::vector<int2> bs_dev;  // (row of bs, device row) of the recorded bias factors whose weights live on the device
};

// Stage 1: the blocks the recorded factors and the old prior touch, which of them are dropped, and their positions:
// dropped blocks, then the dropped inverse depths, then kept blocks (p.n = 0: nothing to marginalize)
int marg_blocks(ctvio_engine* e, MargPlan& p) {
  const ProblemDims d = e->dims();
  const int later = e->opt.ctrl_to_be_opt_later, nowk = e->opt.ctrl_to_be_opt_now;
  const bool drop_knots = later > nowk;  // trajectory_estimator.cpp:161
  p.blocks.assign(d.np, MargBlock());
  bool in_range = true;
  auto touch = [&](int type, int index, bool drop) {
    const int g = ctvio::block_base(type, index, d.nK, d.nB);
    if (g < 0) { in_range = false; return; }
    MargBlock& b = p.blocks[g];
    if (b.type < 0) { b.type = type; b.index = index; }
    b.dropped = b.dropped || drop;
  };
  const ctvio::PriorHost& pr = e->prior;
  if (pr.n > 0) {  // [1] old prior (trajectory_manager.cpp:166-203)
    for (size_t b = 0; b < pr.type.size(); ++b)
      p.use_prior = p.use_prior || ctvio::prior_block_dropped(pr.type[b], pr.index[b], nowk, later);
    if (p.use_prior)
      for (size_t b = 0; b < pr.type.size(); ++b)
        touch(pr.type[b], pr.index[b], ctvio::prior_block_dropped(pr.type[b], pr.index[b], nowk, later));
  }
  // [2] image factors (trajectory_estimator.cpp:325-331), found where the set's structure was built: the knots they
  // touch and two counts.  Their inverse depths are not entered into `blocks`: dropped, they are the last dropped blocks,
  // in landmark order (pos_lm holds their ranks; a device-built set keeps it and marg_img on the device).
  std::vector<uint32_t> knots;
  const int rc = e->n_img_dev > 0 ? marg_discover_device(e, knots, p.n_marg, p.n_rho)
                                  : marg_discover_host(e, knots, p.n_marg, p.n_rho, p.marg_img, p.pos_lm);
  if (rc) return rc;
  for (int kk = 0; kk < e->nK; ++kk)
    if (knots[size_t(kk) / 32] >> (kk % 32) & 1u) {
      touch(CTVIO_BLK_ROT, kk, drop_knots && kk < later);
      touch(CTVIO_BLK_POS, kk, drop_knots && kk < later);
    }
  if (p.n_marg) touch(CTVIO_BLK_LD, 0, false);
  for (size_t k = 0; k < e->imu_order.size(); ++k) {  // [3] IMU factors (:249-257)
    const HostImu& o = e->imu[e->imu_order[k]];
    if (!o.marg) continue;
    p.marg_imu.push_back(int32_t(k));
    const int s = knot_window_first(e, o.t);
    for (int kk = s; kk <= s + 3; ++kk) {
      touch(CTVIO_BLK_ROT, kk, drop_knots && kk < later);
      touch(CTVIO_BLK_POS, kk, drop_knots && kk < later);
    }
    touch(CTVIO_BLK_BG, o.node, true);
    touch(CTVIO_BLK_BA, o.node, true);
  }
  for (size_t k = 0; k < e->biasf.size(); ++k) {  // [4] bias factors (:280-285), drop {bg_i, ba_i}
    const HostBias& o = e->biasf[k];
    if (!o.marg) continue;
    if (int(k) < e->n_bf_dev) p.bs_dev.push_back(make_int2(int(p.bij.size()), int(k)));
    p.bij.push_back(make_int2(o.i, o.j));
    for (int c = 0; c < 6; ++c) p.bs.push_back(o.s[c]);
    touch(CTVIO_BLK_BG, o.i, true); touch(CTVIO_BLK_BG, o.j, false);
    touch(CTVIO_BLK_BA, o.i, true); touch(CTVIO_BLK_BA, o.j, false);
  }
  if (!in_range) return fail(CTVIO_ERR_INVALID, "marginalization block index out of range");

  int pos = 0;
  for (MargBlock& b : p.blocks)
    if (b.type >= 0 && b.dropped) { b.pos = pos; pos += ctvio::block_dim(b.type); }
  pos += p.n_rho;
  p.m = pos;
  for (MargBlock& b : p.blocks)
    if (b.type >= 0 && !b.dropped) { b.pos = pos; pos += ctvio::block_dim(b.type); }
  p.n = pos - p.m;
  p.P = pos;
  if (p.n <= 0) return CTVIO_OK;  // the reference hands back nullptr (trajectory_estimator.cpp:198-201)

  p.pos_cam.assign(d.np, -1);
  for (int g = 0; g < d.np; ++g) {
    const MargBlock& b = p.blocks[g];
    if (b.type >= 0)
      for (int c = 0; c < ctvio::block_dim(b.type); ++c) p.pos_cam[g + c] = b.pos + c;
  }
  p.prior_pos.assign(std::max(pr.n, 1), -1);
  if (p.use_prior)
    for (size_t b = 0; b < pr.type.size(); ++b) {
      const int p0 = p.blocks[ctvio::block_base(pr.type[b], pr.index[b], d.nK, d.nB)].pos;
      for (int c = 0; c < ctvio::block_dim(pr.type[b]); ++c) p.prior_pos[pr.col[b] + c] = p0 + c;
    }
  return CTVIO_OK;
}

// Stage 2: the row-compressed Jacobian of every recorded factor, then [A | b] = Jrow' Jrow in a fixed summation order
int marg_rows(ctvio_engine* e, MargPlan& p) {
  cudaStream_t st = e->stream;
  const ProblemDims d = e->dims();
  ctvio_engine::MargWs& ws = e->mws;
  CUDA_OK(ws.pos_cam.upload(p.pos_cam, st));
  // the landmarks' ranks become positions after the dropped blocks
  if (e->n_img_dev > 0) {
    if (const int rc = offset_pos_lm_device(e, p.m - p.n_rho)) return rc;
  } else {
    for (int32_t& q : p.pos_lm)
      if (q >= 0) q += p.m - p.n_rho;
    CUDA_OK(ws.pos_lm.upload(p.pos_lm, st));
    CUDA_OK(ws.marg_img.upload(p.marg_img, st));
  }
  CUDA_OK(ws.prior_pos.upload(p.prior_pos, st));
  e->n_marg_img = p.n_marg;
  CUDA_OK(ws.marg_imu.upload(p.marg_imu, st));
  CUDA_OK(ws.bij.upload(p.bij, st));
  CUDA_OK(ws.bs.upload(p.bs, st));
  for (const int2 r : p.bs_dev)
    CUDA_OK(cudaMemcpyAsync(ws.bs.p + 6 * size_t(r.x), e->bf_s_dev + 6 * size_t(r.y), 6 * sizeof(double),
                            cudaMemcpyDeviceToDevice, st));
  const int P = p.P;
  CUDA_OK(ws.A.reserve(size_t(P) * P));
  CUDA_OK(ws.b.reserve(P));
  const int n_old = p.use_prior ? e->prior.n : 0;
  const int row_img = 0, row_imu = 2 * p.n_marg, row_bias = row_imu + 6 * int(p.marg_imu.size());
  const int row_prior = row_bias + 6 * int(p.bij.size());
  const int R = row_prior + n_old;
  const int ldj = (P + 2) & ~1;
  CUDA_OK(ws.Jrow.reserve(size_t(std::max(R, 1)) * ldj));
  CUDA_OK(cudaMemsetAsync(ws.Jrow.p, 0, size_t(std::max(R, 1)) * ldj * sizeof(double), st));
  ctvio::MargImageArgs a;
  a.obs = ImageObsPtrs{e->d_img_t.p, e->d_img_pi.p, e->d_img_pj.p, e->d_img_meta.p, int32_t(e->n_img())};
  a.marg_index = ws.marg_img.p; a.n_marg = p.n_marg;
  a.st = e->x[e->cur].ptrs(); a.sp = e->sp; a.rig = e->rig; a.cauchy = e->cfg.cauchy_marg;
  a.pos_cam = ws.pos_cam.p; a.pos_lm = ws.pos_lm.p; a.idx_ld = d.idx_ld;
  a.Jrow = ws.Jrow.p; a.ldj = ldj; a.row0 = row_img; a.P = P; a.scal = e->d_scal.p;
  // the three row kernels write disjoint row ranges of Jrow: one stream each, joined before the SYRK
  cudaEventRecord(e->ev_fork, st);
  e->launches += ctvio::launch_marg_image(a, st);
  ctvio::MargImuArgs b;
  b.obs = ImuObsPtrs{e->d_imu_t.p, e->d_imu_ga.p, int32_t(e->imu.size())};
  b.marg_index = ws.marg_imu.p; b.n_marg = int32_t(p.marg_imu.size());
  b.st = a.st; b.sp = e->sp; b.rig = e->rig; b.pos_cam = ws.pos_cam.p; b.idx_bias0 = d.idx_bias0;
  b.Jrow = ws.Jrow.p; b.ldj = ldj; b.row0 = row_imu; b.P = P; b.scal = e->d_scal.p;
  cudaStreamWaitEvent(e->stream2, e->ev_fork, 0);
  e->launches += ctvio::launch_marg_imu(b, e->stream2);
  cudaEventRecord(e->ev_join, e->stream2);
  ctvio::MargSmallArgs c;
  c.bf_ij = ws.bij.p; c.bf_s = ws.bs.p; c.n_bias = int32_t(p.bij.size());
  c.prior = prior_ptrs(e); c.use_prior = p.use_prior ? 1 : 0; c.prior_pos = ws.prior_pos.p;
  c.st = a.st; c.pos_cam = ws.pos_cam.p; c.idx_bias0 = d.idx_bias0;
  c.Jrow = ws.Jrow.p; c.ldj = ldj; c.row0_bias = row_bias; c.row0_prior = row_prior; c.P = P;
  cudaStreamWaitEvent(e->stream3, e->ev_fork, 0);
  e->launches += ctvio::launch_marg_small(c, e->stream3);
  cudaEventRecord(e->ev_join3, e->stream3);
  cudaStreamWaitEvent(st, e->ev_join, 0);
  cudaStreamWaitEvent(st, e->ev_join3, 0);
  e->launches += ctvio::launch_marg_syrk(ws.Jrow.p, R, ldj, P, ws.A.p, ws.b.p, st);
  return CTVIO_OK;
}

// Stage 3: the dense Schur complement of the m dropped dims through two eigen-decompositions
// (marginalization_factor.cpp:240-263): J_lin, r_lin of the kept n dims in ws.J, ws.r
int marg_schur(ctvio_engine* e, const MargPlan& p) {
  cudaStream_t st = e->stream;
  ctvio_engine::MargWs& ws = e->mws;
  const int m = p.m, n = p.n, P = p.P;
  const double eps = 1e-30;
  auto eig = [&](double* A, double* V, double* ev, int k) {
    const int launched = ctvio::launch_jacobi_eig(A, V, ev, k, ws.eig_scratch.p, st);
    if (launched < 0) return fail(CTVIO_ERR_CUDA, "marginalization: eigen-solver launch refused at n = " + std::to_string(k));
    e->launches += launched;
    return int(CTVIO_OK);
  };
  int rc;
  DevBuf<double>&d_A = ws.A, &d_b = ws.b, &d_Amm = ws.Amm, &d_V = ws.V, &d_ev = ws.ev, &d_Vs = ws.Vs, &d_Ainv = ws.Ainv,
      &d_T = ws.T, &d_Ap = ws.Ap, &d_bp = ws.bp, &d_Ap2 = ws.Ap2, &d_V2 = ws.V2, &d_ev2 = ws.ev2, &d_vb = ws.vb,
      &d_J = ws.J, &d_r = ws.r;
  CUDA_OK(d_Ap.reserve(size_t(n) * n));
  CUDA_OK(d_bp.reserve(n));
  CUDA_OK(cudaMemcpy2DAsync(d_Ap.p, size_t(n) * sizeof(double), d_A.p + size_t(m) * P + m, size_t(P) * sizeof(double),
                            size_t(n) * sizeof(double), n, cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemcpyAsync(d_bp.p, d_b.p + m, size_t(n) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (m > 0) {
    CUDA_OK(d_Amm.reserve(size_t(m) * m)); CUDA_OK(d_V.reserve(size_t(m) * m)); CUDA_OK(d_ev.reserve(m));
    CUDA_OK(d_Vs.reserve(size_t(m) * m)); CUDA_OK(d_Ainv.reserve(size_t(m) * m)); CUDA_OK(d_T.reserve(size_t(n) * m));
    e->launches += ctvio::launch_marg_elementwise(0, m, P, d_A.p, d_Amm.p, nullptr, nullptr, nullptr, eps, st);
    CUDA_OK(ws.eig_scratch.reserve(ctvio::jacobi_log_bytes(std::max(m, n), 40) / sizeof(double) + 1));
    if ((rc = eig(d_Amm.p, d_V.p, d_ev.p, m))) return rc;
    e->launches += ctvio::launch_marg_elementwise(1, m, m, d_V.p, d_Vs.p, d_ev.p, nullptr, nullptr, eps, st);
    e->launches += ctvio::launch_dense_gemm(m, m, m, 1.0, d_Vs.p, m, false, d_V.p, m, true, 0.0, d_Ainv.p, m, st);
    // T = Arm * Amm_inv ; A' = Arr - T * Amr ; b' = brr - T * bmm
    e->launches += ctvio::launch_dense_gemm(n, m, m, 1.0, d_A.p + size_t(m) * P, P, false, d_Ainv.p, m, false, 0.0, d_T.p, m, st);
    e->launches += ctvio::launch_dense_gemm(n, n, m, -1.0, d_T.p, m, false, d_A.p + m, P, false, 1.0, d_Ap.p, n, st);
    e->launches += ctvio::launch_dense_gemm(n, 1, m, -1.0, d_T.p, m, false, d_b.p, 1, false, 1.0, d_bp.p, 1, st);
  }
  CUDA_OK(d_Ap2.reserve(size_t(n) * n)); CUDA_OK(d_V2.reserve(size_t(n) * n)); CUDA_OK(d_ev2.reserve(n));
  CUDA_OK(d_vb.reserve(n)); CUDA_OK(d_J.reserve(size_t(n) * n)); CUDA_OK(d_r.reserve(n));
  e->launches += ctvio::launch_marg_elementwise(2, n, n, d_Ap.p, d_Ap2.p, nullptr, nullptr, nullptr, eps, st);
  CUDA_OK(ws.eig_scratch.reserve(ctvio::jacobi_log_bytes(n, 40) / sizeof(double) + 1));
  if ((rc = eig(d_Ap2.p, d_V2.p, d_ev2.p, n))) return rc;
  e->launches += ctvio::launch_dense_gemm(n, 1, n, 1.0, d_V2.p, n, true, d_bp.p, 1, false, 0.0, d_vb.p, 1, st);
  e->launches += ctvio::launch_marg_elementwise(3, n, n, d_V2.p, d_J.p, d_ev2.p, d_vb.p, d_r.p, eps, st);
  return CTVIO_OK;
}

// Stage 4: the new prior's kept blocks, with the current state as linearisation point.  J_lin / r_lin / x0 STAY in HBM
// (ctvio_adopt_prior hands them over device-to-device, ctvio_get_prior fetches them on demand).
int marg_new_prior(ctvio_engine* e, const MargPlan& p) {
  cudaStream_t st = e->stream;
  ctvio::PriorHost& np_ = e->new_prior;
  np_.n = p.n;
  e->new_prior_on_host = false;
  for (const MargBlock& b : p.blocks) {
    if (b.type < 0 || b.dropped) continue;
    np_.type.push_back(b.type);
    np_.index.push_back(b.index);
    np_.col.push_back(b.pos - p.m);
  }
  DevBuf<int32_t>&d_t = e->mws.new_type, &d_i = e->mws.new_index;
  CUDA_OK(d_t.upload(np_.type, st));
  CUDA_OK(d_i.upload(np_.index, st));
  CUDA_OK(e->d_newprior_x0.reserve(4 * np_.type.size()));
  e->launches += ctvio::launch_prior_x0(e->x[e->cur].ptrs(), d_t.p, d_i.p, int(np_.type.size()), e->d_newprior_x0.p, st);
  CUDA_OK(stream_sync(st));  // the uploads above come from host vectors that are reused by the next call
  return CTVIO_OK;
}

}  // namespace
}  // namespace ctvio::host

// =================================================================================================
extern "C" {

int ctvio_set_prior(ctvio_handle e, int32_t n, const double* J, const double* r, int32_t nb, const int32_t* type,
                    const int32_t* index, const int32_t* col, const double* x0) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  e->prior = ctvio::PriorHost();
  e->prior_dirty = true;
  e->prior_on_device = false;
  e->masks_dirty = true;  // the prior's blocks count as touched parameters
  if (n <= 0) return CTVIO_OK;
  if (!J || !r || nb <= 0 || !type || !index || !col || !x0) return fail(CTVIO_ERR_INVALID, "null argument");
  if (const char* why = ctvio::prior_tiling_error(n, nb, type, col)) return fail(CTVIO_ERR_INVALID, why);
  e->prior.n = n;
  e->prior.J.assign(J, J + size_t(n) * n);
  e->prior.r.assign(r, r + n);
  e->prior.type.assign(type, type + nb);
  e->prior.index.assign(index, index + nb);
  e->prior.col.assign(col, col + nb);
  e->prior.x0.assign(x0, x0 + 4 * size_t(nb));
  return CTVIO_OK;
}

int ctvio_enable_prior(ctvio_handle e, int32_t on) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (e->prior_enabled != (on != 0)) e->masks_dirty = true;
  e->prior_enabled = on != 0;
  return CTVIO_OK;
}

int ctvio_marginalize(ctvio_handle e, int32_t* n_out, int32_t* nb_out) {
  if (!e || !n_out || !nb_out) return fail(CTVIO_ERR_INVALID, "null argument");
  *n_out = 0;
  *nb_out = 0;
  cudaSetDevice(e->cfg.device);
  e->new_prior = ctvio::PriorHost();
  if (!e->opt.is_marg_state) return CTVIO_OK;
  e->n_marg_img = -1;
  ArenaScope arena(e);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  MargPlan p;
  if ((rc = marg_blocks(e, p)) || p.n <= 0) return rc;
  // read_scalars: a recorded factor whose time left its knot window is an error
  if ((rc = marg_rows(e, p)) || (rc = marg_schur(e, p)) || (rc = read_scalars(e)) || (rc = marg_new_prior(e, p))) return rc;
  *n_out = p.n;
  *nb_out = int32_t(e->new_prior.type.size());
  return CTVIO_OK;
}

int ctvio_get_prior(ctvio_handle e, double* J, double* r, int32_t* type, int32_t* index, int32_t* col, double* x0) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (e->new_prior.n <= 0) return fail(CTVIO_ERR_STATE, "no prior has been produced");
  cudaSetDevice(e->cfg.device);
  {
    const int rc = fetch_new_prior(e);
    if (rc) return rc;
  }
  const ctvio::PriorHost& p = e->new_prior;
  if (J) std::memcpy(J, p.J.data(), p.J.size() * sizeof(double));
  if (r) std::memcpy(r, p.r.data(), p.r.size() * sizeof(double));
  if (type) std::memcpy(type, p.type.data(), p.type.size() * sizeof(int32_t));
  if (index) std::memcpy(index, p.index.data(), p.index.size() * sizeof(int32_t));
  if (col) std::memcpy(col, p.col.data(), p.col.size() * sizeof(int32_t));
  if (x0) std::memcpy(x0, p.x0.data(), p.x0.size() * sizeof(double));
  return CTVIO_OK;
}
int ctvio_adopt_prior(ctvio_handle e) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (e->new_prior.n <= 0) return fail(CTVIO_ERR_STATE, "no prior has been produced");
  cudaSetDevice(e->cfg.device);
  return adopt_prior_body(e, false);
}

}  // extern "C"
