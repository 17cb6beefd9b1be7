// Host SVD of the OPQ rounds (index.cu opq_train_device), in a header of its own so that it also builds without CUDA.
#pragma once
#include <algorithm>
#include <cmath>
#include <vector>

namespace gb {
// A (d x d2, row-major) = U diag(s) V^T by one-sided Jacobi on the columns; returns U (d x d2) and V (d2 x d2)
inline void jacobi_svd(std::vector<double>& a, int d, int d2, std::vector<double>* u, std::vector<double>* v) {
  v->assign((size_t)d2 * d2, 0.0);
  for (int i = 0; i < d2; i++) (*v)[(size_t)i * d2 + i] = 1.0;
  for (int sweep = 0; sweep < 60; sweep++) {
    double off = 0;
    for (int p = 0; p < d2 - 1; p++)
      for (int q = p + 1; q < d2; q++) {
        double alpha = 0, beta = 0, gamma = 0;
        for (int i = 0; i < d; i++) {
          const double x = a[(size_t)i * d2 + p], y = a[(size_t)i * d2 + q];
          alpha += x * x, beta += y * y, gamma += x * y;
        }
        if (fabs(gamma) <= 1e-15 * sqrt(alpha * beta) || gamma == 0) continue;
        off = std::max(off, fabs(gamma) / sqrt(alpha * beta + 1e-300));
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
        for (int i = 0; i < d; i++) {
          const double x = a[(size_t)i * d2 + p], y = a[(size_t)i * d2 + q];
          a[(size_t)i * d2 + p] = c * x - sn * y, a[(size_t)i * d2 + q] = sn * x + c * y;
        }
        for (int i = 0; i < d2; i++) {
          const double x = (*v)[(size_t)i * d2 + p], y = (*v)[(size_t)i * d2 + q];
          (*v)[(size_t)i * d2 + p] = c * x - sn * y, (*v)[(size_t)i * d2 + q] = sn * x + c * y;
        }
      }
    if (off < 1e-12) break;
  }
  // U's columns are A V's, normalised.  A column whose norm is at the level of the rotations' rounding noise (d eps
  // times the largest) belongs to a zero singular value and carries no direction: a constant training dimension makes
  // a row of X^T Y exactly 0.  Those columns are completed from an orthonormal basis of the complement of the others,
  // so U stays orthonormal whatever the rank.
  std::vector<double> nrm(d2);
  double nmax = 0;
  for (int j = 0; j < d2; j++) {
    double s = 0;
    for (int i = 0; i < d; i++) s += a[(size_t)i * d2 + j] * a[(size_t)i * d2 + j];
    nrm[j] = sqrt(s);
    nmax = std::max(nmax, nrm[j]);
  }
  const double tol = std::max(d, d2) * 2.220446049250313e-16 * nmax;
  u->assign((size_t)d * d2, 0.0);
  std::vector<int> null_cols;
  for (int j = 0; j < d2; j++) {
    if (nrm[j] > tol) {
      for (int i = 0; i < d; i++) (*u)[(size_t)i * d2 + j] = a[(size_t)i * d2 + j] / nrm[j];
    } else {
      null_cols.push_back(j);
    }
  }
  // each null column: of e_0 .. e_{d-1} with the columns so far projected out (Gram-Schmidt, twice), the one with the
  // largest remainder (its squared norm is at least (d - filled) / d >= 1 / d), normalised.  Unfilled columns are 0.
  std::vector<double> w(d), best(d);
  for (int j : null_cols) {
    double bn = -1;
    for (int e = 0; e < d; e++) {
      std::fill(w.begin(), w.end(), 0.0);
      w[e] = 1.0;
      for (int pass = 0; pass < 2; pass++)
        for (int c = 0; c < d2; c++) {
          double dot = 0;
          for (int i = 0; i < d; i++) dot += (*u)[(size_t)i * d2 + c] * w[i];
          if (dot != 0)
            for (int i = 0; i < d; i++) w[i] -= dot * (*u)[(size_t)i * d2 + c];
        }
      double wn = 0;
      for (int i = 0; i < d; i++) wn += w[i] * w[i];
      if (wn > bn) bn = wn, best = w;
    }
    bn = sqrt(bn);
    for (int i = 0; i < d; i++) (*u)[(size_t)i * d2 + j] = best[i] / bn;
  }
}
}  // namespace gb
