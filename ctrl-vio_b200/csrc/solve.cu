// The LM trust-region driver behind ctvio_solve, its line search and the collectives of sharded mode.
//
// The driver restates Ceres 1.14's TrustRegionMinimizer / LevenbergMarquardtStrategy semantics that
// the reference gets from ceres::Solve (trajectory_estimator.cpp:367-408; SURVEY.md Appendix B):
// Jacobi scaling fixed at iteration 0, D^2 = clamp(diag)/mu, rho = dcost/dmodel accepted above 1e-3,
// mu <- mu / max(1/3, 1-(2rho-1)^3) on success, mu <- mu/f, f <- 2f on failure, function / parameter
// tolerances, Armijo projected line search when the line delay has bounds.
// GPU-first differences from a port: every candidate point is evaluated with full Jacobians into a
// second normal-equation buffer (an accepted step costs no re-linearisation pass), all per-step
// quantities are reduced on the device, and the host reads back ONE 96-byte scalar block per step.
#include <cmath>
#include <cstdlib>

#include "engine_state.h"
#include "poly_min.h"

namespace {

// sharded mode: ONE all-gather of every rank's 8 scalars (sums AND maxima travel together), reduced in a fixed rank
// order by a one-thread kernel that also publishes the common block to mapped host memory (no copy + stream synchronise)
int allreduce_scalars(ctvio_engine* e, bool publish = false) {
  if (e->world <= 1) return CTVIO_OK;
  CUDA_OK(e->d_shard_scal.reserve(8 + 8 * size_t(e->world)));
  e->launches += ctvio::launch_shard_scalars_pack(e->d_scal.p, e->d_shard_scal.p, e->stream);
  std::string err;
  if (!ctvio::comm_allgather(e->nccl_comm, e->d_shard_scal.p, e->d_shard_scal.p + 8, 8, e->stream, &err))
    return fail(CTVIO_ERR_NCCL, err);
  e->launches += ctvio::launch_shard_scalars_reduce(e->d_shard_scal.p + 8, e->world, e->d_scal.p, publish ? e->h_pub : nullptr,
                                                    publish ? ++e->pub_seq : 0, e->stream);
  return CTVIO_OK;
}

// sharded mode: every rank must enter (or skip) the collectives of a solve together.  Sums a per-rank error flag; returns
// CTVIO_OK only if every rank reported local_rc == 0 (a failing rank keeps its own message).
int shard_consensus(ctvio_engine* e, int local_rc) {
  if (e->world <= 1) return local_rc;
  const std::string local_msg = g_err;
  cudaStream_t st = e->stream;
  CUDA_OK(e->d_tmp.reserve(16));
  const double flag = local_rc ? 1.0 : 0.0;
  double total = 0.0;
  CUDA_OK(cudaMemcpyAsync(e->d_tmp.p, &flag, sizeof(double), cudaMemcpyHostToDevice, st));
  std::string err;
  if (!ctvio::comm_allreduce_sum(e->nccl_comm, e->d_tmp.p, 1, st, &err)) return fail(CTVIO_ERR_NCCL, err);
  CUDA_OK(cudaMemcpyAsync(&total, e->d_tmp.p, sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(stream_sync(st));
  if (local_rc) return fail(local_rc, local_msg);
  if (total != 0.0) return fail(CTVIO_ERR_STATE, "another rank of the sharded solve failed before the first collective");
  return CTVIO_OK;
}

// sharded mode: the landmark prologue (hh, the scale of the coupling row) and the per-landmark Schur terms are formed
// from rank-local sums, so all observations of one landmark must live on ONE rank.  Checked once per structure change
// with one all-reduce of the per-landmark owner counts.
int shard_check_ownership(ctvio_engine* e) {
  if (e->world <= 1 || e->shard_checked) return CTVIO_OK;
  cudaStream_t st = e->stream;
  std::vector<double> owned(size_t(std::max(e->nL, 1)), 0.0);
  CUDA_OK(e->d_rho_sync.reserve(2 * size_t(std::max(e->nL, 1))));
  // owned: the landmarks with a factor on this rank (hi > 0 in the built structure)
  CUDA_OK(cudaMemsetAsync(e->d_rho_sync.p, 0, owned.size() * sizeof(double), st));
  if (const int rc = owned_flags_device(e, e->d_rho_sync.p, nullptr)) return rc;
  std::string err;
  if (!ctvio::comm_allreduce_sum(e->nccl_comm, e->d_rho_sync.p, owned.size(), st, &err)) return fail(CTVIO_ERR_NCCL, err);
  CUDA_OK(cudaMemcpyAsync(owned.data(), e->d_rho_sync.p, owned.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(stream_sync(st));
  for (int l = 0; l < e->nL; ++l)
    if (owned[l] > 1.0)
      return fail(CTVIO_ERR_INVALID, "sharded solve: landmark " + std::to_string(l) + " has observations on " +
                                         std::to_string(int(owned[l])) + " ranks (shard image factors by landmark)");
  e->shard_checked = true;
  return CTVIO_OK;
}

// sharded mode: every rank updated only the inverse depths of its own landmark shard: make them consistent everywhere
int shard_sync_inv_depths(ctvio_engine* e) {
  if (e->world <= 1 || e->nL == 0) return CTVIO_OK;
  cudaStream_t st = e->stream;
  CUDA_OK(e->d_rho_sync.reserve(2 * size_t(e->nL)));
  CUDA_OK(e->d_owned.reserve(size_t(e->nL)));
  if (const int rc = owned_flags_device(e, nullptr, e->d_owned.p)) return rc;
  double* rho = e->x[e->cur].rho.p;
  e->launches += ctvio::launch_rho_pack(rho, e->d_owned.p, e->d_rho_sync.p, e->nL, st);
  std::string err;
  if (!ctvio::comm_allreduce_sum(e->nccl_comm, e->d_rho_sync.p, 2 * size_t(e->nL), st, &err)) return fail(CTVIO_ERR_NCCL, err);
  e->launches += ctvio::launch_rho_unpack(rho, e->d_rho_sync.p, e->nL, st);
  return CTVIO_OK;
}

// state update x[to] = x[from] (+) alpha * (dc, dl), line delay clamped into its bounds
ApplyLaunch apply_launch(ctvio_engine* e, int from, int to, double alpha) {
  ApplyLaunch ap;
  ap.dims = e->dims();
  ap.x = e->state(from).ptrs();
  ap.xc = e->state(to).ptrs();
  ap.dc = e->d_dc.p; ap.dl = e->d_dl.p;
  ap.alpha = alpha;
  ap.active = e->d_active.p;
  ap.count_camera = e->rank == 0 ? 1 : 0;
  ap.clamp_ld = e->opt.fix_ld ? 0 : 1;
  ap.ld_lower = e->opt.ld_lower; ap.ld_upper = e->opt.ld_upper;
  ap.scal = e->d_scal.p;
  ap.det_ticket = e->deterministic ? e->d_ticket.p : nullptr;
  return ap;
}

// gradient_norm_kernel at state xb with normal equations nb, the line delay's gradient projected onto its bounds
// publish: the kernel hands the scalar block to mapped host memory (read_scalars(e, true))
// decide: the pipelined driver's device-side step decision; that kernel is chained by programmatic dependent launch
void gradient_norm(ctvio_engine* e, int xb, int nb, bool reset, bool publish, const LmDecideArgs* decide = nullptr) {
  LinearLaunch lin = linear_launch(e, nb);
  lin.pdl = decide ? 1 : 0;
  e->launches += launch_gradient_norm(lin, e->state(xb).ptrs(), e->opt.fix_ld, e->opt.ld_lower, e->opt.ld_upper, e->stream,
                                      reset, publish ? e->h_pub : nullptr, publish ? ++e->pub_seq : 0, decide);
}

// the LM step: reduced system (+ all-reduce of [M | rhs | diagA] over NVLink in sharded mode), factor, solve, and the
// full step applied by ap in the same launch that forms the step vectors
// pdl: the kernels are chained by programmatic dependent launch (pipelined driver only, see launch_chained)
// radius_dev / go: the speculated step reads its radius and go flag from the device-side decision
int lm_step(ctvio_engine* e, int nb, double radius, const ApplyLaunch& ap, bool pdl, const double* radius_dev = nullptr,
            const int32_t* go = nullptr) {
  LinearLaunch lin = linear_launch(e, nb);
  lin.go = go;
  lin.pdl = pdl ? 1 : 0;
  cudaStream_t st = e->stream;
  if (e->deterministic) cudaMemsetAsync(e->d_ticket.p, 0, 2 * sizeof(int32_t), st);
  e->launches += launch_reduced_system(lin, radius, st, radius_dev);
  if (e->world > 1) {
    // one all-reduce of the lower-triangular tiles + rhs + diagonal (half the bytes of the dense slab), damping after it
    std::string err;
    const size_t count = ctvio::shard_pack_len(e->npad);
    CUDA_OK(e->d_shard_pack.reserve(count));
    e->launches += ctvio::launch_shard_pack(lin, e->d_shard_pack.p, st);
    if (!ctvio::comm_allreduce_sum(e->nccl_comm, e->d_shard_pack.p, count, st, &err)) return fail(CTVIO_ERR_NCCL, err);
    e->launches += ctvio::launch_shard_unpack(lin, e->d_shard_pack.p, radius, st);
  }
  e->launches += launch_factor_solve(lin, st);
  e->launches += launch_step_and_apply(lin, ap, st);
  return CTVIO_OK;
}

// zero the normal-equation buffer the NEXT evaluation will accumulate into, on the second stream, so that it overlaps
// the linear solve of this step (only valid when everything enqueued earlier has completed: call right after a read-back)
void prezero_slab(ctvio_engine* e, int nb) {
  cudaMemsetAsync(e->ne_slab[nb].p, 0, e->ne_slab_len * sizeof(double), e->stream2);
  cudaEventRecord(e->ev_zero, e->stream2);
  e->slab_zeroed[nb] = true;
}

// Armijo projected line search (bounds-constrained problems only; Ceres line_search.cc) along the step from x[cur]
// (cost x_cost) to the full-step candidate x[cand], whose scalars are sc.  Leaves the chosen point in x[cand] /
// ne_slab[cand] and its scalars in *e->h_scal; a failed search keeps the full step, as Ceres does.
int line_search(ctvio_engine* e, int cur, int cand, double x_cost, const LmScalars& sc, ctvio_summary& sum) {
  const double ls_sufficient_decrease = 1e-4, ls_max_contraction = 1e-3, ls_min_contraction = 0.6, ls_min_step = 1e-9;
  const int ls_max_iterations = 20;
  cudaStream_t st = e->stream;
  // x[cand] = x[cur] + alpha * step, evaluated with full Jacobians, its scalars read back
  auto evaluate_at = [&](double alpha) {
    if (e->deterministic) cudaMemsetAsync(e->d_ticket.p, 0, 2 * sizeof(int32_t), st);
    e->launches += launch_apply_step(apply_launch(e, cur, cand, alpha), st);
    evaluate(e, cand, cand, true);
    sum.num_jacobian_evals++;
    gradient_norm(e, cand, cand, true, false);
    const int rc = allreduce_scalars(e);
    return rc ? rc : read_scalars(e);
  };
  const double g0 = sc.gd;  // gradient . delta at x
  struct Sample { double x, value, gradient; bool value_ok, grad_ok; };
  Sample initial{0.0, x_cost, g0, true, true}, previous{0, 0, 0, false, false};
  Sample current{1.0, sc.cost_eval, 0.0, std::isfinite(sc.cost_eval), false};
  bool have_grad = false;
  int ls_iters = 0;
  bool success = true;
  while (!current.value_ok || current.value > x_cost + ls_sufficient_decrease * g0 * current.x) {
    ++ls_iters;
    if (ls_iters >= ls_max_iterations) { success = false; break; }
    if (current.value_ok && !have_grad) {
      // directional derivative at the trial point: g(x + a d) . d from the candidate buffers
      e->launches += ctvio::launch_dot_gradient(linear_launch(e, cand), st);
      int rc = allreduce_scalars(e);
      if (rc) return rc;
      rc = read_scalars(e);
      if (rc) return rc;
      current.gradient = e->h_scal->gd;
      current.grad_ok = std::isfinite(current.gradient);
    }
    const double smin = ls_max_contraction * current.x, smax = ls_min_contraction * current.x;
    double step;
    if (!current.value_ok) {
      step = std::min(std::max(current.x * 0.5, smin), smax);
    } else {
      std::vector<ctvio::PolySample> samples;
      samples.push_back({initial.x, initial.value, initial.gradient, true, true});
      samples.push_back({current.x, current.value, current.gradient, true, current.grad_ok});
      if (previous.value_ok) samples.push_back({previous.x, previous.value, previous.gradient, true, previous.grad_ok});
      step = ctvio::minimize_interpolating_polynomial(samples, smin, smax);
    }
    if (step * sc.dir_max < ls_min_step) { success = false; break; }
    previous = current;
    const int rc = evaluate_at(step);
    if (rc) return rc;
    current = Sample{step, e->h_scal->cost_eval, 0.0, std::isfinite(e->h_scal->cost_eval), false};
    have_grad = false;
  }
  sum.num_line_search_steps += ls_iters;
  if (!success && current.x != 1.0) return evaluate_at(1.0);  // rebuild the alpha = 1 candidate
  return CTVIO_OK;
}

// what the host learns from one LM step: from the device-side decision (pipelined driver) or computed on the host
struct StepOutcome {
  bool valid = false;   // the linear solve succeeded and the model decreases
  bool accept = false;  // valid and rho > min_relative_decrease
  double cost = 0, gmax = 0, step_norm2 = 0, x_norm2 = 0;  // at the candidate point
  double radius_next = 0;  // trust-region radius after an accepted step
};

}  // namespace

extern "C" {

int ctvio_solve(ctvio_handle e, int32_t max_iterations, ctvio_summary* out) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  rc = shard_consensus(e, rc);  // every rank leaves here together, or none enters the collectives below
  if (rc) return rc;
  rc = shard_check_ownership(e);
  if (rc) return rc;  // the all-reduced counts are identical on every rank: all of them return
  cudaStream_t st = e->stream;
  const ProblemDims d = e->dims();
  // Ceres 1.14 Solver::Options defaults
  const double initial_radius = 1e4, max_radius = 1e16, min_radius = 1e-32, min_relative_decrease = 1e-3;
  const double function_tolerance = 1e-6, gradient_tolerance = 1e-10, parameter_tolerance = 1e-8;
  const int max_consecutive_invalid = 5;

  ctvio_summary sum;
  std::memset(&sum, 0, sizeof(sum));
  const int64_t launches0 = e->launches;
  cudaEventRecord(e->ev0, st);

  const bool is_constrained = !e->opt.fix_ld && (e->world > 1 || e->h_active[d.idx_ld]);
  if (is_constrained) {  // IterationZero: x = Plus(x, 0) projects the line delay into its bounds
    double ld;
    CUDA_OK(cudaMemcpyAsync(&ld, e->x[e->cur].ld.p, sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_OK(stream_sync(st));
    const double c = std::min(std::max(ld, e->opt.ld_lower), e->opt.ld_upper);
    if (c != ld) CUDA_OK(cudaMemcpyAsync(e->x[e->cur].ld.p, &c, sizeof(double), cudaMemcpyHostToDevice, st));
  }
  ensure_table(e);
  const bool sharded = e->world > 1;
  int cur = e->cur;  // state buffer of the current point
  evaluate(e, cur, cur, true);
  sum.num_jacobian_evals++;
  LinearLaunch lin = linear_launch(e, cur);
  if (sharded) {
    // Jacobi scaling needs the diagonal of the WHOLE camera block: all-reduce it once
    e->launches += launch_extract_diag(lin, st);
    std::string err;
    if (!ctvio::comm_allreduce_sum(e->nccl_comm, lin.diagA, size_t(e->npad), st, &err)) return fail(CTVIO_ERR_NCCL, err);
    e->launches += launch_jacobi_scale_from_diag(lin, st);
  } else {
    e->launches += launch_jacobi_scale(lin, st);
  }
  // (single GPU: published through mapped memory like every later step, no copy + stream synchronisation)
  gradient_norm(e, cur, cur, true, !sharded);
  if (sharded) {
    rc = allreduce_scalars(e);
    if (rc) return rc;
  }
  rc = read_scalars(e, !sharded);
  if (rc) return rc;
  double x_cost = e->h_scal->cost_eval;
  double gmax = e->h_scal->gmax;  // sharded: the all-gathered maximum
  sum.initial_cost = x_cost;
  sum.num_successful_steps = 1;

  double radius = initial_radius, decrease_factor = 2.0;
  int num_invalid = 0;
  bool last_ok = true;
  int iter = 0;
  int term = CTVIO_TERM_NO_CONVERGENCE;

  // Two drivers share the loop below.  The plain one (deterministic mode, sharded mode, a bounded line delay, large
  // windows) takes every step decision on the host.  The pipelined one (single GPU, no bounds, default flush mode)
  // takes the host round trip between two LM steps (publish -> host decision -> launch: a noticeable part of a step at
  // C2) off the critical path: gradient_norm_kernel also takes the accept / radius decision on the device, and the
  // linear solve of step i+1 is enqueued BEFORE the host has seen step i, assuming acceptance (the common case),
  // reading its radius from device memory and writing its candidate into a third state buffer.  When the host then
  // finds step i rejected / invalid / terminating, the speculated kernels' results are simply never used (they touch
  // only the step vectors, the free state buffer and per-step scalars that the next real step resets).
  // It pays at C2 / C5 sizes but was measured slower per LM step at 100 k observations and more, with identical kernels
  // while host timestamps showed the host ahead of the device - cause not found; the round trip it hides is a small
  // part of such a step anyway.  CTVIO_SPECULATION=always / never overrides the size test.
  bool spec_size_ok = e->n_img() <= 20000;
  if (const char* sp = std::getenv("CTVIO_SPECULATION")) {
    if (std::strcmp(sp, "always") == 0) spec_size_ok = true;
    if (std::strcmp(sp, "never") == 0) spec_size_ok = false;
  }
  const bool pipelined = spec_size_ok && !sharded && !is_constrained && !e->deterministic;
  if (pipelined) {
    rc = alloc_state(e, e->xs);
    if (rc) return rc;
  }
  // normal-equation buffer of the current point: flips with the state buffer in the plain driver (cur_ne == cur), on
  // its own in the pipelined one (three state buffers, two normal-equation buffers)
  int cur_ne = cur;
  bool spec_ready = false;      // a speculated linear solve from (cur, cur_ne) into state `spec_out` is in flight
  bool spec_in_flight = false;  // speculated kernels that read ne_slab[cur_ne ^ 1] may still be running
  int spec_out = -1;
  unsigned spec_chol_seq0 = e->chol_seq;
  while (true) {
    if (iter >= max_iterations) { term = CTVIO_TERM_NO_CONVERGENCE; break; }
    if (last_ok && gmax <= gradient_tolerance) { term = CTVIO_TERM_GRADIENT; break; }
    if (radius < min_radius) { term = CTVIO_TERM_MIN_RADIUS; break; }
    ++iter;
    const int cand_ne = cur_ne ^ 1;
    int cand;
    // ---- trust-region step + full evaluation of the candidate ----
    if (spec_ready) {
      cand = spec_out;  // the linear solve of this step already ran (or is running) behind the previous step
      // ne_slab[cand_ne] was the current point's buffer of the previous step: its last reader finished before that
      // step's scalars were published, and the speculated kernels read ne_slab[cur_ne] only
      prezero_slab(e, cand_ne);
    } else {
      cand = 0;
      while (cand == cur) ++cand;
      // everything enqueued so far has completed (scalars were read back): the clear overlaps lm_step; with speculated
      // kernels in flight it is done in stream order by evaluate()
      if (!spec_in_flight) prezero_slab(e, cand_ne);
      // (reduced_system_kernel of lm_step zeroes step_norm2 / x_norm2 / cost_eval / gmax: no memsets on the stream)
      rc = lm_step(e, cur_ne, radius, apply_launch(e, cur, cand, 1.0), pipelined);
      if (rc) return rc;
    }
    sum.num_linear_solves++;
    evaluate(e, cand, cand_ne, true, false);
    sum.num_jacobian_evals++;
    if (pipelined) {
      const LmDecideArgs da{e->d_dec.p, x_cost, radius, min_relative_decrease, max_radius,
                            parameter_tolerance, function_tolerance, gradient_tolerance, min_radius};
      gradient_norm(e, cand, cand_ne, false, true, &da);
      // (no stream operation between this kernel and the speculated reduced_system_kernel: it would cost the two kernels
      // their programmatic dependent launch; ev1 is recorded after the loop, DESIGN §4)
      // ---- speculate: step iter + 1 from (cand, cand_ne), radius from the device-side decision ----
      spec_ready = false;
      if (iter < max_iterations) {
        spec_out = 0;
        while (spec_out == cur || spec_out == cand) ++spec_out;
        spec_chol_seq0 = e->chol_seq;
        rc = lm_step(e, cand_ne, 0.0, apply_launch(e, cand, spec_out, 1.0), true, &e->d_dec.p->radius_next,
                     &e->d_dec.p->go);
        if (rc) return rc;
        spec_ready = true;
        spec_in_flight = true;
      }
    } else {
      // single GPU: the gradient-norm kernel publishes the block; sharded: the reduction kernel behind the all-gather does
      gradient_norm(e, cand, cand_ne, false, !sharded);
      if (sharded) {
        rc = allreduce_scalars(e, true);
        if (rc) return rc;
      }
    }
    rc = read_scalars(e, true);
    if (rc) return rc;
    const LmScalars sc = *e->h_scal;
    StepOutcome o;
    if (pipelined) {
      const LmDecision dec = const_cast<const LmPublished*>(e->h_pub)->dec;
      if (spec_ready && !dec.go) {
        // the device has cancelled the speculated step (its expensive kernels return at once): it does not count as a
        // launch of the tile-DAG solver (message buffer parity), and this driver will not use it.  (go implies a
        // valid, accepted step: a speculated step survives only behind one.)
        e->chol_seq = spec_chol_seq0;
        spec_ready = false;
      }
      if (dec.accept && !spec_ready) spec_in_flight = false;
      o.valid = dec.valid;
      o.accept = dec.accept;
      o.cost = sc.cost_eval; o.gmax = sc.gmax; o.step_norm2 = sc.step_norm2; o.x_norm2 = sc.x_norm2;
      o.radius_next = dec.radius_next;
    } else {
      const double model_cost_change = -sc.gd - 0.5 * sc.dHd;
      o.valid = !sc.chol_fail && std::isfinite(model_cost_change) && model_cost_change > 0.0;
      if (o.valid && is_constrained) {
        rc = line_search(e, cur, cand, x_cost, sc, sum);
        if (rc) return rc;
      }
      const LmScalars& c = *e->h_scal;  // the line search's point, else sc
      o.cost = c.cost_eval; o.gmax = c.gmax; o.step_norm2 = c.step_norm2; o.x_norm2 = c.x_norm2;
      const double rho = (x_cost - o.cost) / model_cost_change;
      o.accept = o.valid && rho > min_relative_decrease;
      o.radius_next = std::min(max_radius, radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * rho - 1.0, 3)));
    }
    // ---- invalid step, tolerances, step acceptance ----
    if (!o.valid) {
      ++sum.num_unsuccessful_steps;
      last_ok = false;
      if (++num_invalid >= max_consecutive_invalid) { term = CTVIO_TERM_FAILURE; break; }
      radius /= decrease_factor;
      decrease_factor *= 2.0;
      continue;
    }
    num_invalid = 0;
    const double step_norm = std::sqrt(o.step_norm2), x_norm = std::sqrt(o.x_norm2);
    if (step_norm <= parameter_tolerance * (x_norm + parameter_tolerance)) { term = CTVIO_TERM_PARAMETER; break; }
    if (std::fabs(x_cost - o.cost) <= function_tolerance * x_cost) { term = CTVIO_TERM_FUNCTION; break; }
    if (o.accept) {
      cur = cand;  // candidate state AND its normal equations become current: no re-linearisation pass
      cur_ne = cand_ne;
      x_cost = o.cost;
      gmax = o.gmax;
      radius = o.radius_next;
      decrease_factor = 2.0;
      last_ok = true;
      ++sum.num_successful_steps;
    } else {
      radius /= decrease_factor;
      decrease_factor *= 2.0;
      last_ok = false;
      ++sum.num_unsuccessful_steps;
    }
  }
  // the current state must live in x[0] / x[1] outside this function: exchange buffer names (kernels in flight hold
  // raw pointers and only touch buffers that are free under either name)
  if (cur == 2) {
    const int f = 0;  // any of the two: neither is current
    DevState &a = e->xs, &b = e->x[f];
    swap(a.q, b.q); swap(a.p, b.p); swap(a.bias, b.bias); swap(a.rho, b.rho); swap(a.ld, b.ld); swap(a.tab, b.tab);
    cur = f;
  }
  e->cur = cur;
  e->table_valid = true;
  e->slab_zeroed[0] = e->slab_zeroed[1] = false;  // (a pending clear is ordered by ev_zero only inside this loop)
  rc = shard_sync_inv_depths(e);
  if (rc) return rc;
  // the timed region of summary.device_ms ends here.  The pipelined driver's last kernels are, when it stopped on a
  // tolerance or a failed step, the speculated step behind the last gradient_norm_kernel, which the device has
  // cancelled (LmDecision::go = 0: its kernels return at once); that tail is included.
  cudaEventRecord(e->ev1, st);
  rc = refresh_mirror(e);  // state -> pinned host mirror, rides on the synchronisation below
  if (rc) return rc;
  CUDA_OK(stream_sync(st));
  float ms = 0;
  cudaEventElapsedTime(&ms, e->ev0, e->ev1);
  sum.iterations = iter;
  sum.termination = term;
  sum.final_cost = x_cost;
  sum.final_radius = radius;
  sum.device_ms = ms;
  sum.kernel_launches = e->launches - launches0;
  if (out) *out = sum;
  return CTVIO_OK;
}

}  // extern "C"
