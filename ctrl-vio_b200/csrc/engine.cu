// Host side of the CUDA engine (the device-resident window's entry points are in resident.cu, the LM trust-region
// driver in solve.cu, the prior and the marginalization in prior.cu): lifecycle, state in / out, factor lists, problem
// preprocessing, evaluation passes, probes and multi-GPU.  Preprocessing is prepare(), a sequence of stages: the image
// structure and the K4 lists (structure.cu, built on the device or on the host), the IMU items, the bias rows, the
// linear-solve buffers, the masks and the prior (prior.cu).
#include <atomic>
#include <cmath>
#include <cstdlib>

#include "engine_state.h"

namespace ctvio::host {

// enqueue the device -> pinned-host copies of the whole state (the caller synchronises the stream afterwards)
int refresh_mirror(ctvio_engine* e) {
  const size_t need = 4 * size_t(e->nK) + kPStride * size_t(e->nK) + 6 * size_t(std::max(e->nB, 1)) + size_t(std::max(e->nL, 1)) + 8;
  if (need > e->h_mirror_cap) {
    if (e->h_mirror) cudaFreeHost(e->h_mirror);
    e->h_mirror = nullptr;
    e->h_mirror_cap = 0;
    if (cudaHostAlloc(reinterpret_cast<void**>(&e->h_mirror), (2 * need) * sizeof(double), cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      e->mirror_valid = false;
      return CTVIO_OK;  // the getters fall back to direct copies
    }
    e->h_mirror_cap = 2 * need;
  }
  DevState& x = e->x[e->cur];
  double* m = e->h_mirror;
  cudaStream_t st = e->stream;
  CUDA_OK(cudaMemcpyAsync(m, x.q.p, 4 * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToHost, st));
  m += 4 * size_t(e->nK);
  CUDA_OK(cudaMemcpyAsync(m, x.p.p, kPStride * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToHost, st));
  m += kPStride * size_t(e->nK);
  if (e->nB) CUDA_OK(cudaMemcpyAsync(m, x.bias.p, 6 * size_t(e->nB) * sizeof(double), cudaMemcpyDeviceToHost, st));
  m += 6 * size_t(std::max(e->nB, 1));
  if (e->nL) CUDA_OK(cudaMemcpyAsync(m, x.rho.p, size_t(e->nL) * sizeof(double), cudaMemcpyDeviceToHost, st));
  m += size_t(std::max(e->nL, 1));
  CUDA_OK(cudaMemcpyAsync(m, x.ld.p, sizeof(double), cudaMemcpyDeviceToHost, st));
  e->mirror_valid = true;  // valid once the caller has synchronised
  return CTVIO_OK;
}

int knot_window_first(const ctvio_engine* e, int64_t t) {
  int64_t s = (t - e->cfg.t0_ns) / e->cfg.dt_ns;
  return int(s);
}

// padded window [first, last] of an evaluation time (se3_spline.h:463-503), clamped to the spline
bool knot_window(const ctvio_engine* e, int64_t t, int& first, int& last) {
  const int64_t maxt = e->cfg.t0_ns + int64_t(e->nK - 3) * e->cfg.dt_ns;
  if (t < e->cfg.t0_ns || t >= maxt) return false;
  const int smax = e->nK - 4;
  const int s1 = knot_window_first(e, t);
  int64_t t2 = t + e->cfg.rs_padding_ns;
  int s2 = (t2 >= maxt) ? smax : int((t2 - e->cfg.t0_ns) / e->cfg.dt_ns);
  if (s2 > s1 + 1) return false;  // padding wider than one knot interval is not supported by the 5-knot window
  first = s1;
  last = std::min(s2 + 3, e->nK - 1);
  return true;
}

// ---- prepare()'s stages (the image structure is built by structure.cu) ----

// IMU samples: sorted into runs of one (start knot, bias node), one CTA each; payload uploaded or gathered on the device
int prepare_imu(ctvio_engine* e) {
  cudaStream_t st = e->stream;
  const int ni = int(e->imu.size());
  std::vector<longlong2> it(ni);
  std::vector<double2> iga(3 * size_t(ni));
  const int64_t maxt = e->cfg.t0_ns + int64_t(e->nK - 3) * e->cfg.dt_ns;
  std::vector<int32_t>& imu_order = e->imu_order;
  imu_order.assign(ni, 0);
  std::vector<int32_t> imu_s(ni);
  for (int k = 0; k < ni; ++k) {
    const HostImu& o = e->imu[k];
    if (o.t < e->cfg.t0_ns || o.t >= maxt) return fail(CTVIO_ERR_TIME_RANGE, "imu time outside the spline");
    if (o.node < 0 || o.node >= e->nB) return fail(CTVIO_ERR_INVALID, "bias node out of range");
    imu_order[k] = k;
    imu_s[k] = knot_window_first(e, o.t);
  }
  // runs of samples sharing (start knot, bias node) -> one CTA each
  std::stable_sort(imu_order.begin(), imu_order.end(), [&](int a, int b) {
    if (imu_s[a] != imu_s[b]) return imu_s[a] < imu_s[b];
    return e->imu[a].node < e->imu[b].node;
  });
  std::vector<ImuItem> imu_items;
  for (int k = 0; k < ni; ++k) {
    const HostImu& o = e->imu[imu_order[k]];
    it[k] = make_longlong2(o.t, o.node);
    iga[3 * k] = make_double2(o.gyro[0], o.gyro[1]);
    iga[3 * k + 1] = make_double2(o.gyro[2], o.accel[0]);
    iga[3 * k + 2] = make_double2(o.accel[1], o.accel[2]);
    const int s = imu_s[imu_order[k]];
    if (imu_items.empty() || imu_items.back().s != s || imu_items.back().node != o.node ||
        imu_items.back().count >= kImuMaxPerItem)
      imu_items.push_back(ImuItem{k, 0, s, o.node});
    imu_items.back().count++;
  }
  e->n_imu_items = int(imu_items.size());
  CUDA_OK(e->d_imu_items.upload(imu_items, st));
  CUDA_OK(e->d_imu_orig.upload(imu_order, st));
  if (!e->imu_src.empty()) {
    // samples taken from the resident IMU table: (table index, bias node) pairs go up, the payload is gathered
    std::vector<int2> src(ni);
    for (int k = 0; k < ni; ++k) src[k] = make_int2(e->imu_src[imu_order[k]], e->imu[imu_order[k]].node);
    CUDA_OK(e->d_imu_src.upload(src, st));
    CUDA_OK(e->d_imu_t.reserve(ni)); CUDA_OK(e->d_imu_ga.reserve(3 * size_t(ni)));
    e->launches += ctvio::launch_gather_imu(e->d_imu_src.p, ni, e->d_imu_tab_t.p, e->d_imu_tab_ga.p, e->d_imu_t.p, e->d_imu_ga.p, st);
  } else {
    CUDA_OK(e->d_imu_t.upload(it, st));
    CUDA_OK(e->d_imu_ga.upload(iga, st));
  }
  return CTVIO_OK;
}

// bias factors: node pairs and sqrt_info rows
int prepare_bias(ctvio_engine* e) {
  cudaStream_t st = e->stream;
  const int nb = int(e->biasf.size());
  std::vector<int2> bij(nb);
  std::vector<double> bs(6 * size_t(nb));
  for (int k = 0; k < nb; ++k) {
    const HostBias& o = e->biasf[k];
    if (o.i < 0 || o.i >= e->nB || o.j < 0 || o.j >= e->nB) return fail(CTVIO_ERR_INVALID, "bias node out of range");
    bij[k] = make_int2(o.i, o.j);
    for (int c = 0; c < 6; ++c) bs[6 * k + c] = o.s[c];
  }
  CUDA_OK(e->d_bf_ij.upload(bij, st));
  if (e->n_bf_dev == 0) {
    CUDA_OK(e->d_bf_s.upload(bs, st));
  } else {
    // rows on the device are copied there; only the host-recorded rows after them go up
    const size_t nd = 6 * size_t(e->n_bf_dev), nh = bs.size() - nd;
    CUDA_OK(e->d_bf_s.reserve(bs.size()));
    CUDA_OK(cudaMemcpyAsync(e->d_bf_s.p, e->bf_s_dev, nd * sizeof(double), cudaMemcpyDeviceToDevice, st));
    if (nh) {
      CUDA_OK(staged_h2d(e->d_bf_s.p + nd, bs.data() + nd, nh * sizeof(double), st));
      g_upload_bytes += nh * sizeof(double);
    }
  }
  return CTVIO_OK;
}

// the normal-equation slabs, the reduced system, the tile-DAG Cholesky's buffers and the solve's vectors
int prepare_linear_buffers(ctvio_engine* e) {
  const ProblemDims d = e->dims();
  const size_t np = size_t(d.np);
  e->off_gc = np * np;
  e->off_hl = e->off_gc + np;
  e->off_gl = e->off_hl + e->nL;
  e->off_wld = e->off_gl + e->nL;
  e->off_W = e->off_wld + e->nL;
  e->ne_slab_len = e->off_W + size_t(e->w_len);
  for (int b = 0; b < 2; ++b) CUDA_OK(e->ne_slab[b].reserve(e->ne_slab_len));
  e->npad = ((d.np + kCholNB - 1) / kCholNB) * kCholNB;
  CUDA_OK(e->d_M.reserve(size_t(e->npad) * e->npad + 3 * size_t(e->npad)));  // M | rhs | diagA | yf (all-reduce slab)
  if (chol_dag_lpub_len(e->npad) > e->d_Linv.cap || chol_dag_part_len(e->npad) > e->d_chol_part.cap || e->linv_npad != e->npad) {
    CUDA_OK(e->d_Linv.reserve(chol_dag_lpub_len(e->npad)));
    CUDA_OK(e->d_chol_part.reserve(chol_dag_part_len(e->npad)));
    e->launches += launch_chol_dag_init(e->d_Linv.p, e->d_chol_part.p, e->npad, e->stream);  // message words start as sentinels
    e->linv_npad = e->npad;
    e->chol_seq = 0;
  }
  if (reduced_system_flags_len(e->npad) > e->d_m_flags.cap) {
    CUDA_OK(e->d_m_flags.reserve(reduced_system_flags_len(e->npad)));
    CUDA_OK(cudaMemsetAsync(e->d_m_flags.p, 0, e->d_m_flags.cap * sizeof(int32_t), e->stream));
  }
  if (chol_dag_flags_len(e->npad) > e->d_chol_flags.cap) {
    CUDA_OK(e->d_chol_flags.reserve(chol_dag_flags_len(e->npad)));
    CUDA_OK(cudaMemsetAsync(e->d_chol_flags.p, 0, e->d_chol_flags.cap * sizeof(int32_t), e->stream));
  }
  CUDA_OK(e->d_y.reserve(e->npad));
  CUDA_OK(e->d_sc.reserve(np));
  CUDA_OK(e->d_sl.reserve(e->nL));
  CUDA_OK(e->d_hh.reserve(e->nL));
  CUDA_OK(e->d_dc.reserve(np));
  CUDA_OK(e->d_dl.reserve(e->nL));
  if (e->nL > 0) CUDA_OK(cudaMemsetAsync(e->d_hh.p, 0, sizeof(double) * e->nL, e->stream));
  return CTVIO_OK;
}

// the constant mask (the options' locked blocks) and the camera part of the active mask (the blocks a factor or the
// prior touches, less the constant ones); the structure build left the landmark part (engine_state.h: h_active)
int prepare_masks(ctvio_engine* e) {
  const ProblemDims d = e->dims();
  e->h_cmask.assign(d.np, 0);
  for (int k = 0; k < e->nK; ++k)
    if (e->opt.lock_traj || (e->opt.fixed_knot_index >= 0 && k <= e->opt.fixed_knot_index))
      for (int c = 0; c < 6; ++c) e->h_cmask[6 * k + c] = 1;  // trajectory_estimator.cpp:134-138
  for (int b = 0; b < e->nB; ++b)
    for (int c = 0; c < 3; ++c) {
      if (e->opt.lock_wb) e->h_cmask[d.idx_bias0 + 6 * b + c] = 1;
      if (e->opt.lock_ab) e->h_cmask[d.idx_bias0 + 6 * b + 3 + c] = 1;
    }
  if (e->opt.fix_ld) e->h_cmask[d.idx_ld] = 1;
  std::vector<uint8_t> touched(d.np, 0);
  auto mark = [&](int f, int l) {
    for (int k = f; k <= l; ++k)
      for (int c = 0; c < 6; ++c) touched[6 * k + c] = 1;
  };
  for (int k = 0; k < e->nK; ++k)  // image factors: the knots of their padded windows, from the structure build
    if (e->img_knots[size_t(k) / 32] >> (k % 32) & 1u) mark(k, k);
  if (e->n_img()) touched[d.idx_ld] = 1;
  for (const HostImu& o : e->imu) {
    const int s = knot_window_first(e, o.t);
    mark(s, s + 3);
    for (int c = 0; c < 6; ++c) touched[d.idx_bias0 + 6 * o.node + c] = 1;
  }
  for (const HostBias& o : e->biasf)
    for (int c = 0; c < 6; ++c) touched[d.idx_bias0 + 6 * o.i + c] = touched[d.idx_bias0 + 6 * o.j + c] = 1;
  if (e->prior.n > 0 && e->prior_enabled)
    for (size_t b = 0; b < e->prior.type.size(); ++b) {
      const int g = ctvio::block_base(e->prior.type[b], e->prior.index[b], d.nK, d.nB);
      if (g >= 0) for (int c = 0; c < ctvio::block_dim(e->prior.type[b]); ++c) touched[g + c] = 1;
    }
  for (int i = 0; i < d.np; ++i) e->h_active[i] = touched[i] && !e->h_cmask[i];
  CUDA_OK(e->d_cmask.upload(e->h_cmask, e->stream));
  CUDA_OK(e->d_active.upload(e->h_active, e->stream));
  e->masks_dirty = false;
  return CTVIO_OK;
}

// Build every structure that depends on the factor set, the sizes or the options, and upload it.
int prepare(ctvio_engine* e) {
  if (!e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  ArenaScope arena(e);
  if (e->nK < 4) return fail(CTVIO_ERR_STATE, "need at least 4 knots");
  if (!e->have_bias) { e->nB = 0; }
  const int T = (e->dims().np + kCholNB - 1) / kCholNB;  // tiles per side of the reduced system (K4 lists)
  // a factor set with table-built factors has its descriptors on the device: its structure is built there
  const bool dev = e->n_img_dev > 0;
  int rc;
  if (e->structure_dirty) {
    e->n_marg_img = -1;  // the last marginalization's block positions describe another structure
    e->shard_checked = false;
    if ((rc = dev ? structure_build_device(e, T) : structure_build_host(e))) return rc;
    if ((rc = prepare_imu(e))) return rc;
    if ((rc = prepare_bias(e))) return rc;
    if ((rc = prepare_linear_buffers(e))) return rc;
    if ((rc = dev ? schur_lists_device(e, T) : schur_lists_host(e, T))) return rc;
    e->prior_dirty = true;
  }
  if ((e->structure_dirty || e->masks_dirty) && (rc = prepare_masks(e))) return rc;
  e->structure_dirty = false;
  if (e->prior_dirty) return prepare_prior(e);
  return CTVIO_OK;
}

VisualLaunch visual_launch(ctvio_engine* e, int xb, int nb, double cauchy) {
  VisualLaunch v;
  v.obs = ImageObsPtrs{e->d_img_t.p, e->d_img_pi.p, e->d_img_pj.p, e->d_img_meta.p, int32_t(e->n_img())};
  v.items = e->d_items.p;
  v.n_items = e->n_items;
  v.st = e->state(xb).ptrs();
  v.ne = e->ne(nb);
  v.lm = e->lml();
  v.dims = e->dims();
  v.sp = e->sp;
  v.rig = e->rig;
  v.cauchy = cauchy;
  v.cmask = e->d_cmask.p;
  v.scal = e->d_scal.p;
  v.det_ticket = e->deterministic ? e->d_ticket.p : nullptr;
  return v;
}
ImuLaunch imu_launch(ctvio_engine* e, int xb, int nb) {
  ImuLaunch v;
  v.obs = ImuObsPtrs{e->d_imu_t.p, e->d_imu_ga.p, int32_t(e->imu.size())};
  v.items = e->d_imu_items.p;
  v.n_items = e->n_imu_items;
  v.st = e->state(xb).ptrs();
  v.ne = e->ne(nb);
  v.dims = e->dims();
  v.sp = e->sp;
  v.rig = e->rig;
  v.cmask = e->d_cmask.p;
  v.scal = e->d_scal.p;
  v.det_ticket = e->deterministic ? e->d_ticket.p : nullptr;
  return v;
}
SmallFactorsLaunch small_launch(ctvio_engine* e, int xb, int nb) {
  SmallFactorsLaunch v;
  v.bf = BiasFactorPtrs{e->d_bf_ij.p, e->d_bf_s.p, int32_t(e->biasf.size())};
  v.prior = prior_ptrs(e);
  v.st = e->state(xb).ptrs();
  v.ne = e->ne(nb);
  v.dims = e->dims();
  v.cmask = e->d_cmask.p;
  v.scal = e->d_scal.p;
  v.deterministic = e->deterministic ? 1 : 0;
  return v;
}
LinearLaunch linear_launch(ctvio_engine* e, int nb) {
  LinearLaunch a;
  a.dims = e->dims();
  a.ne = e->ne(nb);
  a.lm = e->lml();
  a.schur_list = e->d_schur_list.p;
  a.schur_items = e->d_schur_items.p;
  a.n_schur_items = e->n_schur_items;
  a.m_flags = e->d_m_flags.p;
  a.cmask = e->d_cmask.p;
  a.active = e->d_active.p;
  a.sc = e->d_sc.p; a.sl = e->d_sl.p;
  a.M = e->d_M.p; a.Linv = e->d_Linv.p; a.y = e->d_y.p;
  a.rhs = e->d_M.p + size_t(e->npad) * e->npad;
  a.diagA = a.rhs + e->npad;
  a.yf = a.diagA + e->npad;
  a.chol_part = e->d_chol_part.p; a.chol_flags = e->d_chol_flags.p; a.chol_seq = &e->chol_seq;
  a.sharded = e->world > 1 ? 1 : 0;
  a.hh = e->d_hh.p; a.dc = e->d_dc.p; a.dl = e->d_dl.p;
  a.npad = e->npad;
  a.scal = e->d_scal.p;
  a.go = nullptr;
  a.det_ticket = e->deterministic ? e->d_ticket.p : nullptr;
  return a;
}

// one pass over all residual blocks at state buffer xb into normal-equation buffer nb
// reset_cost = false: cost_eval was already zeroed by reduced_system_kernel of the same LM step
void evaluate(ctvio_engine* e, int xb, int nb, bool full, bool reset_cost) {
  cudaStream_t st = e->stream;
  if (full) {
    if (e->slab_zeroed[nb]) {
      cudaStreamWaitEvent(st, e->ev_zero, 0);  // cleared on stream2 while the linear solve was running
      e->slab_zeroed[nb] = false;
    } else {
      cudaMemsetAsync(e->ne_slab[nb].p, 0, e->ne_slab_len * sizeof(double), st);
    }
  }
  if (reset_cost) cudaMemsetAsync(&e->d_scal.p->cost_eval, 0, sizeof(double), st);
  // fork: the (latency-bound) IMU + bias + prior kernels overlap the visual kernel on a second stream
  // sharded mode: IMU / bias / prior factors live on rank 0 only (every rank holds its own landmark shard)
  const bool fork = (e->rank == 0) && (!e->imu.empty() || !e->biasf.empty() || (e->prior.n > 0 && e->prior_enabled));
  if (e->deterministic) {
    // one stream, one kernel at a time, every kernel flushing in block order: every sum has ONE accumulation order
    cudaMemsetAsync(e->d_ticket.p, 0, 2 * sizeof(int32_t), st);
    e->launches += launch_visual(visual_launch(e, xb, nb, e->cfg.cauchy_solve), full, st);
    if (fork) {
      cudaMemsetAsync(e->d_ticket.p, 0, 2 * sizeof(int32_t), st);
      e->launches += launch_imu(imu_launch(e, xb, nb), full, st);
      e->launches += launch_small_factors(small_launch(e, xb, nb), full, st);
    }
    return;
  }
  // (streaming windows: K2 + K3 one after the other take longer than K1 - they get a stream each)
  const bool split = fork && !e->imu.empty() && (!e->biasf.empty() || (e->prior.n > 0 && e->prior_enabled));
  if (fork) {
    cudaEventRecord(e->ev_fork, st);
    cudaStreamWaitEvent(e->stream2, e->ev_fork, 0);
    e->launches += launch_imu(imu_launch(e, xb, nb), full, e->stream2);
    if (split) {
      cudaStreamWaitEvent(e->stream3, e->ev_fork, 0);
      e->launches += launch_small_factors(small_launch(e, xb, nb), full, e->stream3);
      cudaEventRecord(e->ev_join3, e->stream3);
    } else {
      e->launches += launch_small_factors(small_launch(e, xb, nb), full, e->stream2);
    }
    cudaEventRecord(e->ev_join, e->stream2);
  }
  e->launches += launch_visual(visual_launch(e, xb, nb, e->cfg.cauchy_solve), full, st);
  if (fork) cudaStreamWaitEvent(st, e->ev_join, 0);
  if (split) cudaStreamWaitEvent(st, e->ev_join3, 0);
}

// deterministic mode: the flush tickets start at 0 before every ticketed launch (K4 takes [0], the step kernels [1]);
// after an evaluation [0] holds the last factor CTA's value, and a CTA waiting for 0 would spin forever
void reset_tickets(ctvio_engine* e) {
  if (e->deterministic) cudaMemsetAsync(e->d_ticket.p, 0, 2 * sizeof(int32_t), e->stream);
}

// published = true: the last kernel of the step (gradient_norm_kernel) has been asked to write the scalar block to
// mapped host memory with sequence number e->pub_seq: spin on it instead of copy + stream synchronise
int read_scalars(ctvio_engine* e, bool published) {
  if (published) {
    ++g_host_waits;
    volatile unsigned long long* seq = &e->h_pub->seq;
    unsigned spins = 0;
    while (*seq != e->pub_seq) {
      if ((++spins & 0xfffu) == 0 && cudaStreamQuery(e->stream) != cudaErrorNotReady) {
        if (*seq == e->pub_seq) break;
        CUDA_OK(stream_sync(e->stream));
        CUDA_OK(stream_sync(e->stream2));  // (the factor kernels forked onto stream2 are settled too)
        if (*seq != e->pub_seq) return fail(CTVIO_ERR_CUDA, "LM step finished without publishing its scalars");
      }
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    *e->h_scal = const_cast<const LmPublished*>(e->h_pub)->s;
  } else {
    CUDA_OK(cudaMemcpyAsync(e->h_scal, e->d_scal.p, sizeof(LmScalars), cudaMemcpyDeviceToHost, e->stream));
    CUDA_OK(stream_sync(e->stream));
  }
  if ((e->h_scal->error_flags & 1) || (e->world > 1 && e->h_scal->err_sum > 0.0)) {
    cudaMemsetAsync(&e->d_scal.p->error_flags, 0, sizeof(int32_t), e->stream);
    return fail(CTVIO_ERR_TIME_RANGE, "a factor time left its knot window / the spline (line delay too large?)");
  }
  return CTVIO_OK;
}

int add_bias_factors_device(ctvio_engine* e, int n, const int32_t* ni, const int32_t* nj, const double* d_s6,
                            const int32_t* marg) {
  if (int(e->biasf.size()) != e->n_bf_dev) return fail(CTVIO_ERR_STATE, "bias factors with host weights are already present");
  for (int k = 0; k < n; ++k)
    e->biasf.push_back(HostBias{ni[k], nj[k], {0, 0, 0, 0, 0, 0}, marg ? marg[k] : 0});  // weights: d_s6 row k
  e->bf_s_dev = d_s6;
  e->n_bf_dev += n;
  e->structure_dirty = true;
  return CTVIO_OK;
}

int alloc_state(ctvio_engine* e, DevState& s) {
  CUDA_OK(s.q.reserve(4 * size_t(e->nK)));
  CUDA_OK(s.p.reserve(kPStride * size_t(e->nK)));
  CUDA_OK(s.tab.reserve(size_t(std::max(e->nK - 1, 1))));
  CUDA_OK(s.bias.reserve(6 * size_t(std::max(e->nB, 1))));
  CUDA_OK(s.rho.reserve(size_t(std::max(e->nL, 1))));
  CUDA_OK(s.ld.reserve(1));
  return CTVIO_OK;
}

}  // namespace ctvio::host

// =================================================================================================
extern "C" {

const char* ctvio_last_error(void) { return g_err.c_str(); }
int ctvio_abi_version(void) { return CTVIO_ABI_VERSION; }

int ctvio_create(const ctvio_config* cfg, ctvio_handle* out) {
  if (!cfg || !out) return fail(CTVIO_ERR_INVALID, "null argument");
  if (cfg->dt_ns <= 0) return fail(CTVIO_ERR_INVALID, "dt_ns must be positive");
  if (cfg->rs_padding_ns < 0 || cfg->rs_padding_ns > cfg->dt_ns)
    return fail(CTVIO_ERR_INVALID, "rs_padding_ns must lie in [0, dt_ns]: the staged knot window holds 5 knots "
                                   "(4 + one interval of rolling-shutter padding, se3_spline.h:463-503 with 39 ms / 50 ms)");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(CTVIO_ERR_NO_DEVICE, "no CUDA device visible: the ctvio engine has no CPU fallback");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(CTVIO_ERR_NO_DEVICE, "device ordinal out of range");
  CUDA_OK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CUDA_OK(cudaGetDeviceProperties(&prop, cfg->device));
  // sm_90a code runs on compute capability 9.0 only (arch-specific features: no forward compatibility)
  if (prop.major != 9 || prop.minor != 0)
    return fail(CTVIO_ERR_NO_DEVICE, "libctvio_b200 is built for sm_90a (H100) only");
  ctvio_engine* e = new ctvio_engine();
  e->cfg = *cfg;
  std::memset(&e->opt, 0, sizeof(e->opt));
  e->opt.fixed_knot_index = -1;
  e->opt.fix_ld = 1;
  e->sp = SplineParams{cfg->t0_ns, cfg->dt_ns, 0, 1e9 / double(cfg->dt_ns)};
  e->rig.R_CI = so3_matrix(Q4{cfg->q_CtoI[0], cfg->q_CtoI[1], cfg->q_CtoI[2], cfg->q_CtoI[3]});
  e->rig.p_CI = V3{cfg->p_CinI[0], cfg->p_CinI[1], cfg->p_CinI[2]};
  e->rig.w_img = cfg->image_weight;
  e->rig.gravity = V3{cfg->gravity[0], cfg->gravity[1], cfg->gravity[2]};
  for (int k = 0; k < 6; ++k) e->rig.imu_info[k] = cfg->imu_info[k];
  if (const char* det = std::getenv("CTVIO_DETERMINISTIC")) e->deterministic = det[0] == '1';
  if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&e->stream2, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&e->stream3, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_join3, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreate(&e->ev0) != cudaSuccess || cudaEventCreate(&e->ev1) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_join, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&e->ev_zero, cudaEventDisableTiming) != cudaSuccess ||
      e->d_dec.reserve(1) != cudaSuccess ||
      cudaHostAlloc(&e->h_pub, sizeof(LmPublished), cudaHostAllocMapped) != cudaSuccess ||
      cudaMallocHost(&e->h_scal, sizeof(LmScalars)) != cudaSuccess || e->d_scal.reserve(1) != cudaSuccess ||
      e->d_ticket.reserve(4) != cudaSuccess) {
    delete e;
    return fail(CTVIO_ERR_CUDA, "could not create stream / events / scalar block");
  }
  cudaMemsetAsync(e->d_scal.p, 0, sizeof(LmScalars), e->stream);
  std::memset(e->h_pub, 0, sizeof(LmPublished));
  *out = e;
  return CTVIO_OK;
}

int ctvio_destroy(ctvio_handle e) {
  if (!e) return CTVIO_OK;
  cudaSetDevice(e->cfg.device);
  stream_sync(e->stream);
  ctvio::comm_destroy(e->nccl_comm);
  if (e->h_scal) cudaFreeHost(e->h_scal);
  if (e->h_pub) cudaFreeHost(e->h_pub);
  if (e->h_mirror) cudaFreeHost(e->h_mirror);
  if (e->ft.h_map_head) cudaFreeHost(e->ft.h_map_head);
  if (e->cyc.cov_host) cudaFreeHost(e->cyc.cov_host);
  if (e->ckpt.h_stage) cudaFreeHost(e->ckpt.h_stage);
  if (e->ckpt.h_verdict) cudaFreeHost(e->ckpt.h_verdict);
  if (e->ev_zero) cudaEventDestroy(e->ev_zero);
  cudaEventDestroy(e->ev0);
  cudaEventDestroy(e->ev1);
  cudaEventDestroy(e->ev_fork);
  cudaEventDestroy(e->ev_join);
  cudaStreamDestroy(e->stream2);
  if (e->stream3) cudaStreamDestroy(e->stream3);
  if (e->ev_join3) cudaEventDestroy(e->ev_join3);
  cudaStreamDestroy(e->stream);
  delete e;
  return CTVIO_OK;
}

int ctvio_set_options(ctvio_handle e, const ctvio_options* o) {
  if (!e || !o) return fail(CTVIO_ERR_INVALID, "null argument");
  e->opt = *o;
  e->masks_dirty = true;
  e->prior_dirty = true;  // col2g depends on the constant mask
  return CTVIO_OK;
}

int ctvio_set_knots(ctvio_handle e, int32_t n, const double* q, const double* p) {
  if (!e || !q || !p || n < 4) return fail(CTVIO_ERR_INVALID, "need >= 4 knots");
  cudaSetDevice(e->cfg.device);
  if (n != e->nK) e->structure_dirty = true;
  e->nK = n;
  e->sp.n_knots = n;
  for (int b = 0; b < 2; ++b) { const int rc = alloc_state(e, e->x[b]); if (rc) return rc; }
  ArenaScope arena(e);
  std::vector<double> p4(kPStride * size_t(n), 0.0);
  for (int k = 0; k < n; ++k) for (int c = 0; c < 3; ++c) p4[kPStride * k + c] = p[3 * k + c];
  CUDA_OK(staged_h2d(e->x[e->cur].q.p, q, 4 * size_t(n) * sizeof(double), e->stream));
  CUDA_OK(staged_h2d(e->x[e->cur].p.p, p4.data(), p4.size() * sizeof(double), e->stream));  // staged: p4 may go away
  e->mirror_valid = false;
  e->h2d_bytes += size_t(n) * 56;
  e->have_knots = true;
  e->table_valid = false;
  return CTVIO_OK;
}

int ctvio_set_biases(ctvio_handle e, int32_t n, const double* b) {
  if (!e || (n > 0 && !b) || n < 0) return fail(CTVIO_ERR_INVALID, "bad bias array");
  cudaSetDevice(e->cfg.device);
  if (n != e->nB) e->structure_dirty = true;
  e->nB = n;
  for (int k = 0; k < 2; ++k) CUDA_OK(e->x[k].bias.reserve(6 * size_t(std::max(n, 1))));
  ArenaScope arena(e);
  if (n > 0) CUDA_OK(staged_h2d(e->x[e->cur].bias.p, b, 6 * size_t(n) * sizeof(double), e->stream));
  e->mirror_valid = false;
  e->h2d_bytes += size_t(n) * 48;
  e->have_bias = true;
  return CTVIO_OK;
}

int ctvio_set_inv_depths(ctvio_handle e, int32_t n, const double* r) {
  if (!e || (n > 0 && !r) || n < 0) return fail(CTVIO_ERR_INVALID, "bad inverse-depth array");
  cudaSetDevice(e->cfg.device);
  if (n != e->nL) e->structure_dirty = true;
  e->nL = n;
  for (int k = 0; k < 2; ++k) CUDA_OK(e->x[k].rho.reserve(size_t(std::max(n, 1))));
  ArenaScope arena(e);
  if (n > 0) CUDA_OK(staged_h2d(e->x[e->cur].rho.p, r, size_t(n) * sizeof(double), e->stream));
  e->mirror_valid = false;
  e->h2d_bytes += size_t(n) * 8;
  e->have_rho = true;
  return CTVIO_OK;
}

int ctvio_set_time_origin(ctvio_handle e, int64_t t0_ns) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if ((t0_ns - e->cfg.t0_ns) % e->cfg.dt_ns != 0) return fail(CTVIO_ERR_INVALID, "time origin off the knot grid");
  e->cfg.t0_ns = t0_ns;
  e->sp.t0_ns = t0_ns;
  e->structure_dirty = true;
  e->table_valid = false;
  return CTVIO_OK;
}

int ctvio_set_line_delay(ctvio_handle e, double ld) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  cudaSetDevice(e->cfg.device);
  for (int k = 0; k < 2; ++k) CUDA_OK(e->x[k].ld.reserve(1));
  ArenaScope arena(e);
  CUDA_OK(staged_h2d(e->x[e->cur].ld.p, &ld, sizeof(double), e->stream));
  e->mirror_valid = false;
  return CTVIO_OK;
}

int ctvio_get_knots(ctvio_handle e, double* q, double* p) {
  if (!e || !e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  cudaSetDevice(e->cfg.device);
  e->d2h_bytes += size_t(e->nK) * ((q ? 32 : 0) + (p ? 32 : 0));
  if (e->mirror_valid) {  // refreshed by the last solve / re-alignment: no device round trip
    const double* mq = e->h_mirror;
    const double* mp = mq + 4 * size_t(e->nK);
    if (q) std::memcpy(q, mq, 4 * size_t(e->nK) * sizeof(double));
    if (p) for (int k = 0; k < e->nK; ++k) for (int c = 0; c < 3; ++c) p[3 * k + c] = mp[kPStride * k + c];
    return CTVIO_OK;
  }
  if (q) CUDA_OK(cudaMemcpyAsync(q, e->x[e->cur].q.p, 4 * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  std::vector<double> p4;
  if (p) {
    p4.resize(kPStride * size_t(e->nK));
    CUDA_OK(cudaMemcpyAsync(p4.data(), e->x[e->cur].p.p, p4.size() * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  }
  CUDA_OK(stream_sync(e->stream));
  if (p) for (int k = 0; k < e->nK; ++k) for (int c = 0; c < 3; ++c) p[3 * k + c] = p4[kPStride * k + c];
  return CTVIO_OK;
}
int ctvio_get_biases(ctvio_handle e, double* b) {
  if (!e || !b) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  e->d2h_bytes += size_t(e->nB) * 48;
  if (e->mirror_valid) {
    std::memcpy(b, e->h_mirror + (4 + kPStride) * size_t(e->nK), 6 * size_t(e->nB) * sizeof(double));
    return CTVIO_OK;
  }
  if (e->nB > 0) CUDA_OK(cudaMemcpyAsync(b, e->x[e->cur].bias.p, 6 * size_t(e->nB) * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(stream_sync(e->stream));
  return CTVIO_OK;
}
int ctvio_get_inv_depths(ctvio_handle e, double* r) {
  if (!e || !r) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  e->d2h_bytes += size_t(e->nL) * 8;
  if (e->mirror_valid) {
    std::memcpy(r, e->h_mirror + (4 + kPStride) * size_t(e->nK) + 6 * size_t(std::max(e->nB, 1)), size_t(e->nL) * sizeof(double));
    return CTVIO_OK;
  }
  if (e->nL > 0) CUDA_OK(cudaMemcpyAsync(r, e->x[e->cur].rho.p, size_t(e->nL) * sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(stream_sync(e->stream));
  return CTVIO_OK;
}
int ctvio_get_line_delay(ctvio_handle e, double* ld) {
  if (!e || !ld) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  if (e->mirror_valid) {
    *ld = e->h_mirror[(4 + kPStride) * size_t(e->nK) + 6 * size_t(std::max(e->nB, 1)) + size_t(std::max(e->nL, 1))];
    return CTVIO_OK;
  }
  CUDA_OK(cudaMemcpyAsync(ld, e->x[e->cur].ld.p, sizeof(double), cudaMemcpyDeviceToHost, e->stream));
  CUDA_OK(stream_sync(e->stream));
  return CTVIO_OK;
}

int ctvio_clear_factors(ctvio_handle e) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  e->img.clear(); e->imu.clear(); e->biasf.clear();
  e->img_desc.clear(); e->imu_src.clear();
  e->n_img_dev = 0;
  e->n_bf_dev = 0;
  e->structure_dirty = true;
  return CTVIO_OK;
}

int ctvio_add_image_features(ctvio_handle e, int32_t n, const int64_t* ti, const int32_t* rowi, const double* pi,
                             const int64_t* tj, const int32_t* rowj, const double* pj, const int32_t* lm,
                             const int32_t* marg) {
  if (!e || n < 0 || (n > 0 && (!ti || !rowi || !pi || !tj || !rowj || !pj || !lm)))
    return fail(CTVIO_ERR_INVALID, "null argument");
  if (!e->img_desc.empty() || e->n_img_dev > 0)
    return fail(CTVIO_ERR_STATE, "image factors from the resident tables are already present");
  e->img.reserve(e->img.size() + n);
  for (int k = 0; k < n; ++k) {
    HostImage o{ti[k], tj[k], rowi[k], rowj[k], {pi[2 * k], pi[2 * k + 1]}, {pj[2 * k], pj[2 * k + 1]}, lm[k],
                marg ? marg[k] : 0};
    e->img.push_back(o);
  }
  e->structure_dirty = true;
  return CTVIO_OK;
}
int ctvio_add_imu_measurements(ctvio_handle e, int32_t n, const int64_t* t, const double* gyro, const double* accel,
                               const int32_t* node, const int32_t* marg) {
  if (!e || n < 0 || (n > 0 && (!t || !gyro || !accel || !node))) return fail(CTVIO_ERR_INVALID, "null argument");
  if (!e->imu_src.empty()) return fail(CTVIO_ERR_STATE, "IMU factors from the resident table are already present");
  for (int k = 0; k < n; ++k) {
    HostImu o{t[k], {gyro[3 * k], gyro[3 * k + 1], gyro[3 * k + 2]}, {accel[3 * k], accel[3 * k + 1], accel[3 * k + 2]},
              node[k], marg ? marg[k] : 0};
    e->imu.push_back(o);
  }
  e->structure_dirty = true;
  return CTVIO_OK;
}
int ctvio_add_bias_factors(ctvio_handle e, int32_t n, const int32_t* ni, const int32_t* nj, const double* s,
                           const int32_t* marg) {
  if (!e || n < 0 || (n > 0 && (!ni || !nj || !s))) return fail(CTVIO_ERR_INVALID, "null argument");
  for (int k = 0; k < n; ++k) {
    HostBias o{ni[k], nj[k], {s[6 * k], s[6 * k + 1], s[6 * k + 2], s[6 * k + 3], s[6 * k + 4], s[6 * k + 5]},
               marg ? marg[k] : 0};
    e->biasf.push_back(o);
  }
  e->structure_dirty = true;
  return CTVIO_OK;
}

int ctvio_gauge_realign(ctvio_handle e, int32_t min_idx, const double* R0, const double* t0) {
  if (!e || !R0 || !t0 || min_idx < 0 || min_idx >= e->nK) return fail(CTVIO_ERR_INVALID, "bad argument");
  cudaSetDevice(e->cfg.device);
  CUDA_OK(e->d_tmp.reserve(12));
  double h[12];
  for (int k = 0; k < 9; ++k) h[k] = R0[k];
  for (int k = 0; k < 3; ++k) h[9 + k] = t0[k];
  CUDA_OK(cudaMemcpyAsync(e->d_tmp.p, h, sizeof(h), cudaMemcpyHostToDevice, e->stream));  // (stack source: staged by the runtime)
  e->launches += launch_gauge_realign(e->x[e->cur].ptrs(), e->nK, min_idx, e->d_tmp.p, e->stream);
  {
    const int rcm = refresh_mirror(e);
    if (rcm) return rcm;
  }
  CUDA_OK(stream_sync(e->stream));
  e->table_valid = true;
  return CTVIO_OK;
}

int ctvio_save_state(ctvio_handle e) {
  if (!e || !e->have_knots) return fail(CTVIO_ERR_STATE, "state not set");
  cudaSetDevice(e->cfg.device);
  int rc = alloc_state(e, e->snap);
  if (rc) return rc;
  DevState& s = e->x[e->cur];
  cudaStream_t st = e->stream;
  CUDA_OK(cudaMemcpyAsync(e->snap.q.p, s.q.p, 4 * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemcpyAsync(e->snap.p.p, s.p.p, kPStride * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (e->nB) CUDA_OK(cudaMemcpyAsync(e->snap.bias.p, s.bias.p, 6 * size_t(e->nB) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (e->nL) CUDA_OK(cudaMemcpyAsync(e->snap.rho.p, s.rho.p, size_t(e->nL) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemcpyAsync(e->snap.ld.p, s.ld.p, sizeof(double), cudaMemcpyDeviceToDevice, st));
  return CTVIO_OK;
}
int ctvio_restore_state(ctvio_handle e) {
  if (!e || !e->snap.q.p) return fail(CTVIO_ERR_STATE, "no snapshot");
  cudaSetDevice(e->cfg.device);
  DevState& s = e->x[e->cur];
  cudaStream_t st = e->stream;
  CUDA_OK(cudaMemcpyAsync(s.q.p, e->snap.q.p, 4 * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemcpyAsync(s.p.p, e->snap.p.p, kPStride * size_t(e->nK) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (e->nB) CUDA_OK(cudaMemcpyAsync(s.bias.p, e->snap.bias.p, 6 * size_t(e->nB) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  if (e->nL) CUDA_OK(cudaMemcpyAsync(s.rho.p, e->snap.rho.p, size_t(e->nL) * sizeof(double), cudaMemcpyDeviceToDevice, st));
  CUDA_OK(cudaMemcpyAsync(s.ld.p, e->snap.ld.p, sizeof(double), cudaMemcpyDeviceToDevice, st));
  e->table_valid = false;
  e->mirror_valid = false;
  return CTVIO_OK;
}

// ---- probes --------------------------------------------------------------------------------------
int ctvio_eval_image_factors(ctvio_handle e, int32_t want_jac, double cauchy, double* r, int32_t* s, double* J,
                             double* cost) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  const size_t n = e->n_img();
  DevBuf<double> dr, dJ;
  DevBuf<int32_t> ds;
  CUDA_OK(dr.reserve(2 * n));
  CUDA_OK(ds.reserve(2 * n));
  if (want_jac) CUDA_OK(dJ.reserve(100 * n));
  cudaStream_t st = e->stream;
  cudaMemsetAsync(&e->d_scal.p->cost_eval, 0, sizeof(double), st);
  e->launches += launch_probe_image(visual_launch(e, e->cur, e->cur, cauchy), e->d_img_orig.p, want_jac != 0, dr.p, ds.p,
                                    want_jac ? dJ.p : nullptr, st);
  rc = read_scalars(e);
  if (rc) return rc;
  if (r && n) CUDA_OK(cudaMemcpy(r, dr.p, 2 * n * sizeof(double), cudaMemcpyDeviceToHost));
  if (s && n) CUDA_OK(cudaMemcpy(s, ds.p, 2 * n * sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (J && want_jac && n) CUDA_OK(cudaMemcpy(J, dJ.p, 100 * n * sizeof(double), cudaMemcpyDeviceToHost));
  if (cost) *cost = e->h_scal->cost_eval;
  return CTVIO_OK;
}

int ctvio_eval_imu_factors(ctvio_handle e, int32_t want_jac, double* r, int32_t* s, double* J, double* cost) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  const size_t n = e->imu.size();
  DevBuf<double> dr, dJ;
  DevBuf<int32_t> ds;
  CUDA_OK(dr.reserve(6 * n));
  CUDA_OK(ds.reserve(n));
  if (want_jac) CUDA_OK(dJ.reserve(156 * n));
  cudaStream_t st = e->stream;
  cudaMemsetAsync(&e->d_scal.p->cost_eval, 0, sizeof(double), st);
  e->launches += launch_probe_imu(imu_launch(e, e->cur, e->cur), e->d_imu_orig.p, want_jac != 0, dr.p, ds.p,
                                  want_jac ? dJ.p : nullptr, st);
  rc = read_scalars(e);
  if (rc) return rc;
  if (r && n) CUDA_OK(cudaMemcpy(r, dr.p, 6 * n * sizeof(double), cudaMemcpyDeviceToHost));
  if (s && n) CUDA_OK(cudaMemcpy(s, ds.p, n * sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (J && want_jac && n) CUDA_OK(cudaMemcpy(J, dJ.p, 156 * n * sizeof(double), cudaMemcpyDeviceToHost));
  if (cost) *cost = e->h_scal->cost_eval;
  return CTVIO_OK;
}

int ctvio_residual_summary(ctvio_handle e, int32_t* counts, double* sums, double* prior_sum) {
  if (!e || !counts || !sums) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  cudaStream_t st = e->stream;
  const size_t ni = e->n_img(), nm = e->imu.size(), nb = e->biasf.size();
  const int np_ = e->prior_enabled ? e->prior.n : 0;
  DevBuf<double> dr, dout;
  DevBuf<int32_t> ds;
  CUDA_OK(dr.reserve(2 * ni + 6 * nm + 8));
  CUDA_OK(ds.reserve(2 * ni + nm + 8));
  CUDA_OK(dout.reserve(18));
  CUDA_OK(cudaMemsetAsync(dout.p, 0, 18 * sizeof(double), st));
  // residuals without the loss (cauchy scale 0 = no corrector), original factor order does not matter for the sums
  if (ni) e->launches += launch_probe_image(visual_launch(e, e->cur, e->cur, 0.0), e->d_img_orig.p, false, dr.p, ds.p, nullptr, st);
  if (nm) e->launches += launch_probe_imu(imu_launch(e, e->cur, e->cur), e->d_imu_orig.p, false, dr.p + 2 * ni, ds.p + 2 * ni, nullptr, st);
  e->launches += ctvio::launch_abs_column_sums(dr.p, int(ni), 2, dout.p, st);
  e->launches += ctvio::launch_abs_column_sums(dr.p + 2 * ni, int(nm), 6, dout.p + 2, st);
  e->launches += ctvio::launch_bias_abs_sums(e->d_bf_ij.p, e->d_bf_s.p, int(nb), e->x[e->cur].bias.p, dout.p + 8, st);
  if (np_ > 0) {
    e->launches += launch_small_factors(small_launch(e, e->cur, e->cur), false, st);  // leaves r + J dx in prior.res
  }
  rc = read_scalars(e);
  if (rc) return rc;
  CUDA_OK(cudaMemcpy(sums, dout.p, 18 * sizeof(double), cudaMemcpyDeviceToHost));
  counts[0] = int32_t(ni); counts[1] = int32_t(nm); counts[2] = int32_t(nb); counts[3] = np_ > 0 ? 1 : 0;
  if (prior_sum && np_ > 0) {
    CUDA_OK(cudaMemcpy(prior_sum, e->d_prior_res.p, size_t(np_) * sizeof(double), cudaMemcpyDeviceToHost));
    for (int i = 0; i < np_; ++i) prior_sum[i] = std::fabs(prior_sum[i]);
  }
  return CTVIO_OK;
}

int ctvio_eval_cost(ctvio_handle e, double* cost) {
  if (!e || !cost) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  evaluate(e, e->cur, e->cur, false);
  rc = read_scalars(e);
  if (rc) return rc;
  *cost = e->h_scal->cost_eval;
  return CTVIO_OK;
}

int ctvio_normal_equations(ctvio_handle e, double* Hcc, double* gc, double* hl, double* gl, double* cost) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  evaluate(e, e->cur, e->cur, true);
  rc = read_scalars(e);
  if (rc) return rc;
  const ProblemDims d = e->dims();
  const size_t np = d.np;
  NormalEqPtrs ne = e->ne(e->cur);
  if (Hcc) {
    std::vector<double> up(np * np);
    CUDA_OK(cudaMemcpy(up.data(), ne.A, np * np * sizeof(double), cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < np; ++i)
      for (size_t j = i; j < np; ++j) Hcc[i * np + j] = Hcc[j * np + i] = up[i * np + j];
  }
  if (gc) CUDA_OK(cudaMemcpy(gc, ne.gc, np * sizeof(double), cudaMemcpyDeviceToHost));
  if (hl && e->nL) CUDA_OK(cudaMemcpy(hl, ne.hl, e->nL * sizeof(double), cudaMemcpyDeviceToHost));
  if (gl && e->nL) CUDA_OK(cudaMemcpy(gl, ne.gl, e->nL * sizeof(double), cudaMemcpyDeviceToHost));
  if (cost) *cost = e->h_scal->cost_eval;
  return CTVIO_OK;
}

int ctvio_query_trajectory(ctvio_handle e, int32_t n, const int64_t* t, double* q, double* p, double* omega,
                           double* vel, double* acc) {
  if (!e || n < 0 || (n > 0 && !t)) return fail(CTVIO_ERR_INVALID, "bad argument");
  if (!e->have_knots) return fail(CTVIO_ERR_STATE, "knots have not been set");
  cudaSetDevice(e->cfg.device);
  ensure_table(e);
  if (n == 0) return CTVIO_OK;
  DevBuf<int64_t> dt;
  DevBuf<double> out;
  CUDA_OK(dt.reserve(n));
  CUDA_OK(out.reserve(16 * size_t(n)));
  cudaStream_t st = e->stream;
  CUDA_OK(cudaMemcpyAsync(dt.p, t, size_t(n) * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  QueryLaunch a;
  a.st = e->x[e->cur].ptrs();
  a.sp = e->sp;
  a.n = n;
  a.t = dt.p;
  a.q = out.p; a.p = out.p + 4 * size_t(n); a.omega = out.p + 7 * size_t(n); a.vel = out.p + 10 * size_t(n);
  a.acc = out.p + 13 * size_t(n);
  a.scal = e->d_scal.p;
  e->launches += launch_query(a, st);
  int rc = read_scalars(e);
  if (rc) return rc;
  if (q) CUDA_OK(cudaMemcpy(q, a.q, 4 * size_t(n) * sizeof(double), cudaMemcpyDeviceToHost));
  if (p) CUDA_OK(cudaMemcpy(p, a.p, 3 * size_t(n) * sizeof(double), cudaMemcpyDeviceToHost));
  if (omega) CUDA_OK(cudaMemcpy(omega, a.omega, 3 * size_t(n) * sizeof(double), cudaMemcpyDeviceToHost));
  if (vel) CUDA_OK(cudaMemcpy(vel, a.vel, 3 * size_t(n) * sizeof(double), cudaMemcpyDeviceToHost));
  if (acc) CUDA_OK(cudaMemcpy(acc, a.acc, 3 * size_t(n) * sizeof(double), cudaMemcpyDeviceToHost));
  return CTVIO_OK;
}

int ctvio_profile_kernels(ctvio_handle e, int32_t reps, int32_t flush_l2, double* out) {
  if (!e || !out || reps == 0) return fail(CTVIO_ERR_INVALID, "bad argument");
  const bool visual_only = reps < 0;  // reps < 0: only out_ms[0] (K1) - usable on a sharded engine (no collectives)
  if (visual_only) reps = -reps;
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  cudaStream_t st = e->stream;
  const int cur = e->cur, cand = cur ^ 1;
  DevBuf<unsigned char> flush;
  const size_t flush_bytes = size_t(256) << 20;
  if (flush_l2) CUDA_OK(flush.reserve(flush_bytes));
  if (visual_only) {
    for (int k = 0; k < 8; ++k) out[k] = 0.0;
    double total = 0;
    for (int it = -3; it < reps; ++it) {
      if (flush_l2) cudaMemsetAsync(flush.p, it & 0xff, flush_bytes, st);
      cudaMemsetAsync(e->ne_slab[cur].p, 0, e->ne_slab_len * sizeof(double), st);
      reset_tickets(e);
      cudaEventRecord(e->ev0, st);
      launch_visual(visual_launch(e, cur, cur, e->cfg.cauchy_solve), true, st);
      cudaEventRecord(e->ev1, st);
      if (cudaEventSynchronize(e->ev1) != cudaSuccess) return fail(CTVIO_ERR_CUDA, "kernel failed while profiling");
      float ms = 0;
      cudaEventElapsedTime(&ms, e->ev0, e->ev1);
      if (it >= 0) total += ms;
    }
    out[0] = total / reps;
    cudaMemsetAsync(&e->d_scal.p->error_flags, 0, sizeof(int32_t), st);
    CUDA_OK(stream_sync(st));
    return CTVIO_OK;
  }
  // a valid linearisation + step so that every stage has meaningful inputs
  evaluate(e, cur, cur, true);
  LinearLaunch lin = linear_launch(e, cur);
  launch_jacobi_scale(lin, st);
  reset_tickets(e);
  launch_lm_step(lin, 1e4, st);
  rc = read_scalars(e);
  if (rc) return rc;
  ApplyLaunch ap;
  ap.dims = e->dims();
  ap.x = e->x[cur].ptrs(); ap.xc = e->x[cand].ptrs();
  ap.dc = e->d_dc.p; ap.dl = e->d_dl.p; ap.alpha = 1.0; ap.active = e->d_active.p;
  ap.count_camera = 1;
  ap.clamp_ld = e->opt.fix_ld ? 0 : 1; ap.ld_lower = e->opt.ld_lower; ap.ld_upper = e->opt.ld_upper;
  ap.scal = e->d_scal.p;
  auto time_stage = [&](int stage, double* ms_out) -> int {
    double total = 0;
    for (int it = -3; it < reps; ++it) {
      if (flush_l2) cudaMemsetAsync(flush.p, it & 0xff, flush_bytes, st);
      if (stage == 0 || stage == 1 || stage == 2)
        cudaMemsetAsync(e->ne_slab[cur].p, 0, e->ne_slab_len * sizeof(double), st);
      reset_tickets(e);
      cudaEventRecord(e->ev0, st);
      switch (stage) {
        case 0: launch_visual(visual_launch(e, cur, cur, e->cfg.cauchy_solve), true, st); break;
        case 1: launch_imu(imu_launch(e, cur, cur), true, st); break;
        case 2: launch_small_factors(small_launch(e, cur, cur), true, st); break;
        case 3: launch_reduced_system(lin, 1e4, st); break;
        case 4: launch_factor_solve(lin, st); break;
        case 5: launch_step_vectors(lin, st); break;
        case 6: launch_apply_step(ap, st); break;
        default: launch_visual(visual_launch(e, cur, cur, e->cfg.cauchy_solve), false, st); break;
      }
      cudaEventRecord(e->ev1, st);
      if (cudaEventSynchronize(e->ev1) != cudaSuccess) return fail(CTVIO_ERR_CUDA, "kernel failed while profiling");
      float ms = 0;
      cudaEventElapsedTime(&ms, e->ev0, e->ev1);
      if (it >= 0) total += ms;
    }
    *ms_out = total / reps;
    return CTVIO_OK;
  };
  // stage order keeps inputs valid: 3 (reduced system) must precede 4 (it is factored in place)
  for (int stage : {0, 1, 2, 7}) { rc = time_stage(stage, &out[stage]); if (rc) return rc; }
  evaluate(e, cur, cur, true);  // restore a complete set of normal equations
  {
    double total3 = 0, total4 = 0, total5 = 0;
    for (int it = -3; it < reps; ++it) {
      float ms;
      if (flush_l2) cudaMemsetAsync(flush.p, it & 0xff, flush_bytes, st);
      reset_tickets(e);  // (both: K4 takes [0], the step kernels below [1])
      cudaEventRecord(e->ev0, st); launch_reduced_system(lin, 1e4, st); cudaEventRecord(e->ev1, st);
      cudaEventSynchronize(e->ev1); cudaEventElapsedTime(&ms, e->ev0, e->ev1); if (it >= 0) total3 += ms;
      if (flush_l2) cudaMemsetAsync(flush.p, it & 0xff, flush_bytes, st);
      cudaEventRecord(e->ev0, st); launch_factor_solve(lin, st); cudaEventRecord(e->ev1, st);
      cudaEventSynchronize(e->ev1); cudaEventElapsedTime(&ms, e->ev0, e->ev1); if (it >= 0) total4 += ms;
      if (flush_l2) cudaMemsetAsync(flush.p, it & 0xff, flush_bytes, st);
      cudaEventRecord(e->ev0, st); launch_step_vectors(lin, st); cudaEventRecord(e->ev1, st);
      cudaEventSynchronize(e->ev1); cudaEventElapsedTime(&ms, e->ev0, e->ev1); if (it >= 0) total5 += ms;
    }
    out[3] = total3 / reps; out[4] = total4 / reps; out[5] = total5 / reps;
  }
  rc = time_stage(6, &out[6]);
  if (rc) return rc;
  cudaMemsetAsync(&e->d_scal.p->error_flags, 0, sizeof(int32_t), st);
  CUDA_OK(stream_sync(st));
  return CTVIO_OK;
}

int ctvio_selfcheck_solver(ctvio_handle e, int32_t reps, int32_t* mismatches, double* rel_residual) {
  if (!e || !mismatches || !rel_residual || reps <= 0) return fail(CTVIO_ERR_INVALID, "bad argument");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  ensure_table(e);
  cudaStream_t st = e->stream;
  const int cur = e->cur;
  evaluate(e, cur, cur, true);
  LinearLaunch lin = linear_launch(e, cur);
  launch_jacobi_scale(lin, st);
  reset_tickets(e);
  launch_reduced_system(lin, 1e4, st);
  const size_t n = size_t(e->npad), len = n * n + n;  // M | rhs are contiguous
  DevBuf<double> backup;
  CUDA_OK(backup.reserve(len));
  CUDA_OK(cudaMemcpyAsync(backup.p, lin.M, len * sizeof(double), cudaMemcpyDeviceToDevice, st));
  std::vector<double> hM(len), x0(n), x(n);
  CUDA_OK(cudaMemcpyAsync(hM.data(), lin.M, len * sizeof(double), cudaMemcpyDeviceToHost, st));
  *mismatches = 0;
  for (int r = 0; r < reps; ++r) {
    if (r > 0) CUDA_OK(cudaMemcpyAsync(lin.M, backup.p, len * sizeof(double), cudaMemcpyDeviceToDevice, st));
    launch_factor_solve(lin, st);
    CUDA_OK(cudaMemcpyAsync((r == 0 ? x0 : x).data(), lin.y, n * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_OK(stream_sync(st));
    if (r > 0 && std::memcmp(x.data(), x0.data(), n * sizeof(double)) != 0) ++*mismatches;
  }
  // residual of the first solve against the host copy (only the lower triangle of M is maintained by K4)
  for (size_t i = 0; i < n; ++i)
    for (size_t j = i + 1; j < n; ++j) hM[i * n + j] = hM[j * n + i];
  const double* rhs = hM.data() + n * n;
  double rmax = 0, bmax = 0;
  for (size_t i = 0; i < n; ++i) {
    double s = -rhs[i];
    for (size_t j = 0; j < n; ++j) s += hM[i * n + j] * x0[j];
    rmax = std::max(rmax, std::fabs(s));
    bmax = std::max(bmax, std::fabs(rhs[i]));
  }
  *rel_residual = bmax > 0 ? rmax / bmax : rmax;
  cudaMemsetAsync(&e->d_scal.p->error_flags, 0, sizeof(int32_t), st);
  CUDA_OK(stream_sync(st));
  return CTVIO_OK;
}

// Test hook (not part of include/ctvio.h): the stages of one LM step at the current state, with the launchers lm_step
// uses (K6 as the separate step-vector kernel: the state is not updated), and every stage's inputs and outputs copied
// to `out`.  *len: capacity of `out` in doubles on entry, the length needed on return (out == nullptr: query only).
// Layout, np = 6 (nK + nB) + 1, npad = np rounded up to 64, all row-major doubles:
//   header[16]  np, npad, nL, K4 work items, gd, dHd, dir_max, chol_fail, 0...
//   A[np][np] (upper triangle valid, unscaled) | gc[np] | hl[nL] | gl[nL] | W[nL][np] (dense; wld in column np - 1)
//   | cmask[np] (1 = constant) | sc[np] | sl[nL] | hh[nL]           -- what K4 reads (hh: written by K4)
//   | M[npad][npad] (lower triangle valid) | rhs[npad]             -- K4's output, before K5 factors M in place
//   | y[npad]                                                         -- K5
//   | dc[np] | dl[nL]                                                 -- K6
// poison != 0: M and rhs are filled with NaN before K4 runs, so that an entry K4 fails to write shows in the output.
int ctvio_debug_lm_step_poison(ctvio_handle e, double radius, double* out, int64_t* len, int32_t poison) {
  if (!e || !len || !(radius > 0.0)) return fail(CTVIO_ERR_INVALID, "bad argument");
  cudaSetDevice(e->cfg.device);
  int rc = prepare(e);
  if (rc) return rc;
  const ProblemDims d = e->dims();
  const size_t np = size_t(d.np), nL = size_t(e->nL), npad = size_t(e->npad);
  const size_t need = 16 + np * np + np + 2 * nL + nL * np + 2 * np + 2 * nL + npad * npad + 2 * npad + np + nL;
  const int64_t cap = *len;
  *len = int64_t(need);
  if (!out) return CTVIO_OK;
  if (cap < int64_t(need)) return fail(CTVIO_ERR_INVALID, "output slab too small");
  ensure_table(e);
  cudaStream_t st = e->stream;
  const int cur = e->cur;
  evaluate(e, cur, cur, true);
  rc = read_scalars(e);
  if (rc) return rc;
  LinearLaunch lin = linear_launch(e, cur);
  launch_jacobi_scale(lin, st);
  reset_tickets(e);
  if (poison) CUDA_OK(cudaMemsetAsync(lin.M, 0xff, (npad * npad + npad) * sizeof(double), st));  // M | rhs: all-ones NaN
  launch_reduced_system(lin, radius, st);
  double* o = out + 16;
  double* A = o; o += np * np;
  double* gc = o; o += np;
  double* hl = o; o += nL;
  double* gl = o; o += nL;
  double* W = o; o += nL * np;
  double* cm = o; o += np;
  double* sc = o; o += np;
  double* sl = o; o += nL;
  double* hh = o; o += nL;
  double* M = o; o += npad * npad;
  double* rhs = o; o += npad;
  double* y = o; o += npad;
  double* dc = o; o += np;
  double* dl = o;
  // (pageable destinations: each copy has completed when it returns, so M and rhs are taken before K5 runs)
  CUDA_OK(cudaMemcpyAsync(M, lin.M, npad * npad * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(rhs, lin.rhs, npad * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(stream_sync(st));
  launch_factor_solve(lin, st);
  CUDA_OK(cudaMemcpyAsync(y, lin.y, npad * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(stream_sync(st));
  launch_step_vectors(lin, st);
  const NormalEqPtrs ne = e->ne(cur);
  std::vector<double> Wc(size_t(e->w_len)), wld(nL);
  std::vector<uint8_t> hm(np);
  std::vector<int32_t> lo(nL), hi(nL);  // the landmark layout, read back (a device-built structure has no host copy)
  std::vector<int64_t> woff(nL);
  CUDA_OK(cudaMemcpyAsync(A, ne.A, np * np * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(gc, ne.gc, np * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(hm.data(), lin.cmask, np, cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(sc, lin.sc, np * sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_OK(cudaMemcpyAsync(dc, lin.dc, np * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (nL) {
    CUDA_OK(cudaMemcpyAsync(hl, ne.hl, nL * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpyAsync(gl, ne.gl, nL * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpyAsync(wld.data(), ne.wld, nL * sizeof(double), cudaMemcpyDeviceToHost, st));
    if (!Wc.empty()) CUDA_OK(cudaMemcpyAsync(Wc.data(), ne.W, Wc.size() * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpyAsync(sl, lin.sl, nL * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpyAsync(hh, lin.hh, nL * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpyAsync(dl, lin.dl, nL * sizeof(double), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpyAsync(lo.data(), e->d_lo.p, nL * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpyAsync(hi.data(), e->d_hi.p, nL * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaMemcpyAsync(woff.data(), e->d_woff.p, nL * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  }
  CUDA_OK(cudaMemcpyAsync(e->h_scal, e->d_scal.p, sizeof(LmScalars), cudaMemcpyDeviceToHost, st));
  cudaMemsetAsync(&e->d_scal.p->error_flags, 0, sizeof(int32_t), st);
  CUDA_OK(stream_sync(st));
  std::memset(W, 0, nL * np * sizeof(double));
  for (size_t l = 0; l < nL; ++l) {
    for (int g = lo[l]; g < hi[l]; ++g) W[l * np + g] = Wc[size_t(woff[l]) + (g - lo[l])];
    W[l * np + size_t(d.idx_ld)] = wld[l];
  }
  for (size_t i = 0; i < np; ++i) cm[i] = hm[i] ? 1.0 : 0.0;
  const LmScalars& s = *e->h_scal;
  std::memset(out, 0, 16 * sizeof(double));
  out[0] = double(np); out[1] = double(npad); out[2] = double(nL); out[3] = double(e->n_schur_items);
  out[4] = s.gd; out[5] = s.dHd; out[6] = s.dir_max; out[7] = double(s.chol_fail);
  return CTVIO_OK;
}
int ctvio_debug_lm_step(ctvio_handle e, double radius, double* out, int64_t* len) {
  return ctvio_debug_lm_step_poison(e, radius, out, len, 0);
}

int ctvio_measure_fp64_tflops(ctvio_handle e, double* tflops) {
  if (!e || !tflops) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  const double v = ctvio::measure_fp64_tflops(e->stream);
  if (v < 0) return fail(CTVIO_ERR_CUDA, "fp64 micro-benchmark failed");
  *tflops = v;
  return CTVIO_OK;
}

int ctvio_measure_fp64_tensor_tflops(ctvio_handle e, double* tflops) {
  if (!e || !tflops) return fail(CTVIO_ERR_INVALID, "null argument");
  cudaSetDevice(e->cfg.device);
  const double v = ctvio::measure_fp64_tensor_tflops(e->stream);
  if (v < 0) return fail(CTVIO_ERR_CUDA, "fp64 tensor-core micro-benchmark failed");
  *tflops = v;
  return CTVIO_OK;
}

int ctvio_set_deterministic(ctvio_handle e, int32_t on) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (e->world > 1 && on) return fail(CTVIO_ERR_STATE, "deterministic mode is single-GPU");
  e->deterministic = on != 0;
  e->structure_dirty = true;  // K1 work items are rebuilt with single-round chunks
  return CTVIO_OK;
}

int ctvio_sync_stats(ctvio_handle e, int64_t* host_waits, int32_t reset) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (host_waits) *host_waits = g_host_waits;
  if (reset) g_host_waits = 0;
  return CTVIO_OK;
}

int ctvio_transfer_stats(ctvio_handle e, int64_t* h2d_bytes, int64_t* d2h_bytes, int32_t reset) {
  if (!e) return fail(CTVIO_ERR_INVALID, "null handle");
  if (h2d_bytes) *h2d_bytes = int64_t(e->h2d_bytes + g_upload_bytes);
  if (d2h_bytes) *d2h_bytes = int64_t(e->d2h_bytes);
  if (reset) { e->h2d_bytes = e->d2h_bytes = 0; g_upload_bytes = 0; }
  return CTVIO_OK;
}

int ctvio_nccl_unique_id(uint8_t* id128) {
  if (!id128) return fail(CTVIO_ERR_INVALID, "null argument");
  std::string err;
  if (!ctvio::comm_unique_id(id128, &err)) return fail(CTVIO_ERR_NCCL, err);
  return CTVIO_OK;
}
int ctvio_comm_init(ctvio_handle e, int32_t rank, int32_t world, const uint8_t* id128) {
  if (!e || !id128 || world < 1 || rank < 0 || rank >= world) return fail(CTVIO_ERR_INVALID, "bad argument");
  cudaSetDevice(e->cfg.device);
  std::string err;
  void* comm = ctvio::comm_create(rank, world, id128, &err);
  if (!comm) return fail(CTVIO_ERR_NCCL, err);
  ctvio::comm_destroy(e->nccl_comm);
  e->nccl_comm = comm;
  e->rank = rank;
  e->world = world;
  e->shard_checked = false;
  return CTVIO_OK;
}

}  // extern "C"
