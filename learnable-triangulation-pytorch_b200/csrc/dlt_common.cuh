// The float64 eigen-solve of the DLT triangulations: the weighted DLT of the algebraic model (algebraic.cu) and the RANSAC
// triangulation (ransac.cu) accumulate their own rows into M = A^T A and share this one solver.
#pragma once
#include <math.h>

namespace lt {

// M = A^T A diagonalised by cyclic Jacobi rotations: on return M's diagonal holds the eigenvalues, the columns of E the
// eigenvectors, and the result is the index of the smallest eigenvalue (the first one on a tie).
__host__ __device__ __forceinline__ int dlt_jacobi(double M[4][4], double E[4][4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) E[r][c] = r == c ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 16; ++sweep) {
    double off = 0.0;
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int q = p + 1; q < 4; ++q) off += M[p][q] * M[p][q];
    if (off < 1e-300) break;
#pragma unroll
    for (int p = 0; p < 4; ++p) {
#pragma unroll
      for (int q = p + 1; q < 4; ++q) {
        if (M[p][q] == 0.0) continue;
        const double theta = (M[q][q] - M[p][p]) / (2.0 * M[p][q]);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
        for (int k = 0; k < 4; ++k) { const double a = M[k][p], bb = M[k][q]; M[k][p] = c * a - s * bb; M[k][q] = s * a + c * bb; }
#pragma unroll
        for (int k = 0; k < 4; ++k) { const double a = M[p][k], bb = M[q][k]; M[p][k] = c * a - s * bb; M[q][k] = s * a + c * bb; }
#pragma unroll
        for (int k = 0; k < 4; ++k) { const double a = E[k][p], bb = E[k][q]; E[k][p] = c * a - s * bb; E[k][q] = s * a + c * bb; }
      }
    }
  }
  // compile-time indices only (the select loops below too): M and E stay in registers
  int m = 0;
  double lm = M[0][0];
#pragma unroll
  for (int k = 1; k < 4; ++k)
    if (M[k][k] < lm) { lm = M[k][k]; m = k; }
  return m;
}

// u = column m of E
__host__ __device__ __forceinline__ void dlt_column(const double E[4][4], int m, double u[4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    u[r] = E[r][0];
#pragma unroll
    for (int k = 1; k < 4; ++k)
      if (k == m) u[r] = E[r][k];
  }
}

}  // namespace lt
