// ORACLE (test infrastructure, NOT product code).  Parity unpinned (see so3.hpp).
// Window problem, normal equations, Ceres-1.14-style LM loop and VINS-style
// marginalization restated on the CPU in fp64.
//
// Restates:
//   estimator/trajectory_estimator.cpp:114-141  AddControlPoints (constant knots)
//   estimator/trajectory_estimator.cpp:143-204  Prepare/SaveMarginalizationInfo
//   estimator/trajectory_estimator.cpp:219-348  Add*Factor (block lists, drop sets, losses)
//   estimator/trajectory_estimator.cpp:367-408  Solve -> ceres::Solve options
//   factor/analytic_diff/marginalization_factor.cpp:85-265  marginalize()
//   spline/se3_spline.h:463-503                  CaculateSplineMeta (padded knot windows)
//   estimator/trajectory_manager.cpp:485-516     double2vector (4-DoF gauge re-alignment)
//   Ceres-Solver 1.14 (NOT part of the reference repository; pinned only by README.md:15):
//     trust_region_minimizer.cc, levenberg_marquardt_strategy.cc, line_search.cc,
//     polynomial.cc, corrector.cc, loss_function.cc, parameter_block.h  — restated
//     from the published algorithm (SURVEY.md Appendix B).
#pragma once
#include <cstdint>
#include <vector>

#include "factors.hpp"

namespace ctvio_oracle {

struct Options {
  int fixed_knot_index = -1;  // SetFixedIndex (trajectory_estimator.h:90)
  bool lock_traj = false;
  bool lock_wb = false, lock_ab = false;
  bool fix_ld = true;
  double ld_lower = 0.0, ld_upper = 0.0;
  int64_t rs_padding_ns = 39000000;  // trajectory_estimator.cpp:299
  double cauchy_solve = 2.0, cauchy_marg = 1.0;  // :321
  bool is_marg_state = false;
  int ctrl_to_be_opt_now = 0, ctrl_to_be_opt_later = 0;
  int num_threads = 1;
};

enum Termination { kNoConvergence = 0, kConvergenceGradient = 1, kConvergenceParameter = 2,
                   kConvergenceFunction = 3, kFailure = 4, kMinRadius = 5 };

struct Summary {
  int iterations = 0;  // accepted + rejected (+ invalid) steps after iteration 0
  int num_successful_steps = 0, num_unsuccessful_steps = 0;
  int termination = kNoConvergence;
  double initial_cost = 0, final_cost = 0;
  int num_cost_evals = 0;      // cost-only passes over all residual blocks
  int num_jacobian_evals = 0;  // residual+Jacobian passes (incl. line-search gradient passes)
  int num_linear_solves = 0;
  int num_line_search_steps = 0;
  double final_radius = 0;
  double t_eval_s = 0, t_schur_s = 0, t_solve_s = 0, t_total_s = 0;
};

// Schur-form normal equations at a linearisation point.
struct NormalEq {
  int nK = 0, nB = 0, nL = 0, np = 0;
  double cost = 0;
  std::vector<double> Hcc;  // np x np row-major (upper triangle filled, symmetrised on demand)
  std::vector<double> gc;   // np
  std::vector<double> hl, gl, wld;  // per landmark: diag, gradient, coupling to line delay
  std::vector<int> lo, hi;          // per landmark camera-dim range [lo, hi) (knot dims)
  std::vector<size_t> woff;         // nL + 1
  std::vector<double> W;            // per landmark coupling over [lo, hi)
};

class Window {
 public:
  SplineGrid grid;
  Calib cal;
  Options opt;
  std::vector<double> q, p;   // knots [nK][4], [nK][3]
  std::vector<double> bias;   // [nB][6]  (bg, ba)
  std::vector<double> rho;    // [nL]
  double ld = 0.0;
  std::vector<ImageObs> img;
  std::vector<ImuObs> imu;
  std::vector<BiasObs> biasf;
  Prior prior;      // prior used by solve()
  Prior new_prior;  // produced by marginalize()

  int nK() const { return int(q.size() / 4); }
  int nB() const { return int(bias.size() / 6); }
  int nL() const { return int(rho.size()); }
  int np() const { return 6 * nK() + 6 * nB() + 1; }
  int idxKnot(int k) const { return 6 * k; }
  int idxBias(int b) const { return 6 * nK() + 6 * b; }
  int idxLd() const { return 6 * nK() + 6 * nB(); }

  enum Mode { kCost = 0, kGradient = 1, kFull = 2 };
  // Evaluate all residual blocks at the current state.
  double assemble(Mode mode, NormalEq* ne) const;
  Summary solve(int max_iterations);
  bool marginalize();
  // trajectory_manager.cpp:485-516; R0/t0 are the pre-solve pose of knot min_idx.
  void gauge_realign(int min_idx, const double R0[9], const double t0[3]);

  // padded knot window [first, last] of an evaluation at time t (se3_spline.h:463-503)
  void knotWindow(int64_t t, int& first, int& last) const;
  void buildStructure(NormalEq* ne) const;
  std::vector<char> constMask() const;   // np flags
  std::vector<char> touchedMask() const; // np flags + landmarks appended
};

}  // namespace ctvio_oracle
