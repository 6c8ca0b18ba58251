// Step-size selection of the Armijo line search that Ceres 1.14 runs inside its trust-region loop
// when a parameter has bounds (the camera line delay, trajectory_estimator.cpp:314-318):
// interpolate cost (and directional derivative) samples with a polynomial and minimise it on
// [x_min, x_max] (Ceres internal/ceres/polynomial.cc; Ceres is not part of the reference repository).
// Host-only, a few flops per LM step.
#pragma once
#include <algorithm>
#include <cmath>
#include <complex>
#include <vector>

namespace ctvio {

struct PolySample {
  double x, value, gradient;
  bool value_ok, gradient_ok;
};

namespace polydetail {
inline double horner(const std::vector<double>& c, double x) {  // highest degree first
  double v = 0;
  for (double a : c) v = v * x + a;
  return v;
}
// Gaussian elimination with complete pivoting (Eigen fullPivLu in Ceres)
inline std::vector<double> solve(std::vector<double> A, std::vector<double> b) {
  const int n = int(b.size());
  std::vector<int> perm(n);
  for (int i = 0; i < n; ++i) perm[i] = i;
  for (int k = 0; k < n; ++k) {
    int pr = k, pc = k;
    double best = -1;
    for (int i = k; i < n; ++i)
      for (int j = k; j < n; ++j)
        if (std::fabs(A[i * n + j]) > best) { best = std::fabs(A[i * n + j]); pr = i; pc = j; }
    if (!(best > 0)) break;
    for (int j = 0; j < n; ++j) std::swap(A[k * n + j], A[pr * n + j]);
    std::swap(b[k], b[pr]);
    for (int i = 0; i < n; ++i) std::swap(A[i * n + k], A[i * n + pc]);
    std::swap(perm[k], perm[pc]);
    for (int i = k + 1; i < n; ++i) {
      const double f = A[i * n + k] / A[k * n + k];
      for (int j = k; j < n; ++j) A[i * n + j] -= f * A[k * n + j];
      b[i] -= f * b[k];
    }
  }
  std::vector<double> y(n, 0.0), x(n, 0.0);
  for (int i = n - 1; i >= 0; --i) {
    double s = b[i];
    for (int j = i + 1; j < n; ++j) s -= A[i * n + j] * y[j];
    y[i] = A[i * n + i] != 0 ? s / A[i * n + i] : 0.0;
  }
  for (int i = 0; i < n; ++i) x[perm[i]] = y[i];
  return x;
}
// real parts of all roots of a polynomial (Ceres evaluates the candidates at the real parts of complex
// roots too)
inline std::vector<double> root_real_parts(std::vector<double> c) {
  while (c.size() > 1 && c.front() == 0.0) c.erase(c.begin());
  const int deg = int(c.size()) - 1;
  std::vector<double> out;
  if (deg <= 0) return out;
  if (deg == 1) { out.push_back(-c[1] / c[0]); return out; }
  if (deg == 2) {
    const double a = c[0], b = c[1], cc = c[2];
    const double D = b * b - 4 * a * cc, sD = std::sqrt(std::fabs(D));
    if (D >= 0) {
      if (b >= 0) { out.push_back((-b - sD) / (2 * a)); out.push_back((2 * cc) / (-b - sD)); }
      else { out.push_back((2 * cc) / (-b + sD)); out.push_back((-b + sD) / (2 * a)); }
    } else {
      out.push_back(-b / (2 * a)); out.push_back(-b / (2 * a));
    }
    return out;
  }
  using cd = std::complex<double>;
  std::vector<cd> m(deg + 1);
  for (int i = 0; i <= deg; ++i) m[i] = c[i] / c[0];
  double bound = 0;
  for (int i = 1; i <= deg; ++i) bound = std::max(bound, std::abs(m[i]));
  bound += 1.0;
  std::vector<cd> z(deg);
  for (int i = 0; i < deg; ++i) z[i] = std::polar(0.5 * bound, 2.0 * M_PI * i / deg + 0.4);
  for (int it = 0; it < 500; ++it) {  // Durand-Kerner
    double change = 0;
    for (int i = 0; i < deg; ++i) {
      cd num = 0, den = 1;
      for (int k = 0; k <= deg; ++k) num = num * z[i] + m[k];
      for (int j = 0; j < deg; ++j) if (j != i) den *= (z[i] - z[j]);
      if (std::abs(den) == 0) den = 1e-300;
      const cd dz = num / den;
      z[i] -= dz;
      change = std::max(change, std::abs(dz));
    }
    if (change < 1e-15 * bound) break;
  }
  for (const cd& r : z) out.push_back(r.real());
  return out;
}
}  // namespace polydetail

inline double minimize_interpolating_polynomial(const std::vector<PolySample>& samples, double x_min, double x_max) {
  int nc = 0;
  for (const PolySample& s : samples) nc += int(s.value_ok) + int(s.gradient_ok);
  const int deg = nc - 1;
  std::vector<double> lhs(size_t(nc) * nc, 0.0), rhs(nc, 0.0);
  int row = 0;
  for (const PolySample& s : samples) {
    if (s.value_ok) {
      for (int j = 0; j <= deg; ++j) lhs[row * nc + j] = std::pow(s.x, deg - j);
      rhs[row++] = s.value;
    }
    if (s.gradient_ok) {
      for (int j = 0; j < deg; ++j) lhs[row * nc + j] = (deg - j) * std::pow(s.x, deg - j - 1);
      rhs[row++] = s.gradient;
    }
  }
  const std::vector<double> poly = polydetail::solve(lhs, rhs);
  double best_x = 0.5 * (x_min + x_max), best_v = polydetail::horner(poly, best_x);
  auto consider = [&](double x) {
    const double v = polydetail::horner(poly, x);
    if (v < best_v) { best_v = v; best_x = x; }
  };
  consider(x_min);
  consider(x_max);
  if (poly.size() > 2) {
    std::vector<double> dpoly(deg);
    for (int i = 0; i < deg; ++i) dpoly[i] = (deg - i) * poly[i];
    for (double r : polydetail::root_real_parts(dpoly))
      if (r >= x_min && r <= x_max) consider(r);
  }
  for (const PolySample& s : samples)
    if (s.x >= x_min && s.x <= x_max && s.value_ok && s.value < best_v) { best_v = s.value; best_x = s.x; }
  return best_x;
}

}  // namespace ctvio
