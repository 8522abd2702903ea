// Calibrated multi-view geometry of the labeled training step (lightning-pose 3-D mode).
//   pairwise triangulation     lightning_pose/data/cameras.py:22-83   (kornia undistort_points + triangulate_points)
//   3-D -> 2-D projection      lightning_pose/data/cameras.py:86-171  (kornia PinholeCamera.project + distort_points)
//   frame -> model coordinates lightning_pose/data/bboxes.py:194-219  (frame_to_model_batch)
//   pairwise-projection loss   lightning_pose/losses/losses.py:999-1126
//
// Design notes: the reference loops in Python over batch x camera pairs, gathers valid keypoints with boolean masks and
// backpropagates through torch.linalg.svd; every mask and its `torch.any(has_distortion)` branch is a host sync.  Here
// one thread owns one small problem (a pair's DLT, a point's projection into every view) and decides NaN / distortion
// on the device.  The per-thread geometry runs in fp64: the DLT goes through M = A^T A, which squares the condition
// number, and calibrations with focal lengths of 1e5 are in use.  Backward kernels recompute the forward (a few hundred
// flops per point) instead of keeping a workspace; each input gradient is summed by one thread in a fixed order, so
// gradients are bit-identical run to run.  No atomics anywhere.
#include <cstdint>

#include "../../include/lpb200.h"
#include "lpb_common.cuh"

namespace lpb {
namespace {

constexpr int CAM_THREADS = 128;
constexpr int CAM_MAX_VIEWS = 64;
constexpr int UNDISTORT_ITERS = 5;  // kornia undistort_points(num_iters=5)
constexpr int JACOBI_SWEEPS = 10;   // cyclic Jacobi on a 4x4 symmetric matrix: converged to fp64 rounding in <= 6
constexpr double HOMOG_EPS = 1e-8;  // kornia convert_points_from_homogeneous(eps=1e-8)

// OpenCV / kornia distortion coefficients, zero-padded to 12 (k1 k2 p1 p2 k3 k4 k5 k6 s1 s2 s3 s4); `any`: the row is
// not all zero (the reference's per-(batch, view) has_distortion, cameras.py:149)
struct Dist {
  double k1, k2, p1, p2, k3, k4, k5, k6, s1, s2, s3, s4;
  bool any;
};

__device__ __forceinline__ Dist load_dist(const float* __restrict__ d, int P) {
  double c[12];
  bool any = false;
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    const float v = i < P ? d[i] : 0.f;
    c[i] = v;
    any |= (v != 0.f);
  }
  return Dist{c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7], c[8], c[9], c[10], c[11], any};
}

// pinhole intrinsics as the distortion model reads them (fx, fy, cx, cy; skew ignored)
struct Pinhole {
  double fx, fy, cx, cy;
};
__device__ __forceinline__ Pinhole load_pinhole(const float* __restrict__ K) { return Pinhole{K[0], K[4], K[2], K[5]}; }

__device__ __forceinline__ double homog_scale(double z) { return fabs(z) > HOMOG_EPS ? 1.0 / (z + HOMOG_EPS) : 1.0; }

// ---- undistortion: kornia undistort_points with new_K = I (fixed-point iterations in normalised coordinates) --------
__device__ __forceinline__ void undistort_step(const Dist& d, double x0, double y0, double x, double y, double& xn, double& yn) {
  const double r2 = x * x + y * y;
  const double inv = (1.0 + d.k4 * r2 + d.k5 * r2 * r2 + d.k6 * r2 * r2 * r2) / (1.0 + d.k1 * r2 + d.k2 * r2 * r2 + d.k3 * r2 * r2 * r2);
  const double dx = 2.0 * d.p1 * x * y + d.p2 * (r2 + 2.0 * x * x) + d.s1 * r2 + d.s2 * r2 * r2;
  const double dy = d.p1 * (r2 + 2.0 * y * y) + 2.0 * d.p2 * x * y + d.s3 * r2 + d.s4 * r2 * r2;
  xn = (x0 - dx) * inv;
  yn = (y0 - dy) * inv;
}

// adjoint of one iteration at its input (x, y): (gxn, gyn) on its output -> (gx, gy) on (x, y), accumulated into (gx0, gy0)
__device__ __forceinline__ void undistort_step_adj(const Dist& d, double x0, double y0, double x, double y, double gxn, double gyn,
                                                   double& gx, double& gy, double& gx0, double& gy0) {
  const double r2 = x * x + y * y;
  const double N = 1.0 + d.k4 * r2 + d.k5 * r2 * r2 + d.k6 * r2 * r2 * r2, dN = d.k4 + 2.0 * d.k5 * r2 + 3.0 * d.k6 * r2 * r2;
  const double D = 1.0 + d.k1 * r2 + d.k2 * r2 * r2 + d.k3 * r2 * r2 * r2, dD = d.k1 + 2.0 * d.k2 * r2 + 3.0 * d.k3 * r2 * r2;
  const double q = N / D, dq = (dN * D - N * dD) / (D * D);
  const double dx = 2.0 * d.p1 * x * y + d.p2 * (r2 + 2.0 * x * x) + d.s1 * r2 + d.s2 * r2 * r2;
  const double dy = d.p1 * (r2 + 2.0 * y * y) + 2.0 * d.p2 * x * y + d.s3 * r2 + d.s4 * r2 * r2;
  const double ts = d.s1 + 2.0 * d.s2 * r2, tt = d.s3 + 2.0 * d.s4 * r2;
  const double dx_x = 2.0 * d.p1 * y + 6.0 * d.p2 * x + 2.0 * x * ts, dx_y = 2.0 * d.p1 * x + 2.0 * d.p2 * y + 2.0 * y * ts;
  const double dy_x = 2.0 * d.p1 * x + 2.0 * d.p2 * y + 2.0 * x * tt, dy_y = 6.0 * d.p1 * y + 2.0 * d.p2 * x + 2.0 * y * tt;
  const double gr2 = (gxn * (x0 - dx) + gyn * (y0 - dy)) * dq;
  gx = -(gxn * dx_x + gyn * dy_x) * q + 2.0 * x * gr2;
  gy = -(gxn * dx_y + gyn * dy_y) * q + 2.0 * y * gr2;
  gx0 += gxn * q;
  gy0 += gyn * q;
}

// pixel (u, v) -> undistorted normalised (x, y); xs / ys (optional) receive the input of every iteration
__device__ __forceinline__ void undistort(const Pinhole& c, const Dist& d, double u, double v, double& x, double& y,
                                          double* xs = nullptr, double* ys = nullptr) {
  const double x0 = (u - c.cx) / c.fx, y0 = (v - c.cy) / c.fy;
  x = x0;
  y = y0;
#pragma unroll
  for (int i = 0; i < UNDISTORT_ITERS; ++i) {
    if (xs) {
      xs[i] = x;
      ys[i] = y;
    }
    undistort_step(d, x0, y0, x, y, x, y);
  }
}

// reverse mode through the recorded iterations: gradient on the undistorted point -> gradient on the pixel
__device__ __forceinline__ void undistort_adj(const Pinhole& c, const Dist& d, const double* xs, const double* ys, double gx,
                                              double gy, double& gu, double& gv) {
  const double x0 = xs[0], y0 = ys[0];
  double gx0 = 0.0, gy0 = 0.0;
#pragma unroll
  for (int i = UNDISTORT_ITERS - 1; i >= 0; --i) {
    double nx, ny;
    undistort_step_adj(d, x0, y0, xs[i], ys[i], gx, gy, nx, ny, gx0, gy0);
    gx = nx;
    gy = ny;
  }
  gu = (gx0 + gx) / c.fx;  // the first iterate is x0 itself
  gv = (gy0 + gy) / c.fy;
}

// ---- DLT: smallest eigenvector of M = A^T A by cyclic Jacobi ----------------------------------------------------------
struct Dlt {
  double A[4][4];
  double U[4][4];  // eigenvectors (columns)
  double lam[4];   // eigenvalues
  double lmin;     // the smallest one
  int imin;
  double v[4];     // U[:, imin], sign fixed so that v[3] >= 0
};

// one Jacobi rotation zeroing a[p][q]: a <- J^T a J, U <- U J
template <int p, int q>
__device__ __forceinline__ void jacobi_rotate(double (&a)[4][4], double (&U)[4][4]) {
  const double apq = a[p][q];
  if (apq == 0.0) return;
  const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
  const double t = copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
  const double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double akp = a[k][p], akq = a[k][q];
    a[k][p] = cs * akp - sn * akq;
    a[k][q] = sn * akp + cs * akq;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double apk = a[p][k], aqk = a[q][k];
    a[p][k] = cs * apk - sn * aqk;
    a[q][k] = sn * apk + cs * aqk;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const double ukp = U[k][p], ukq = U[k][q];
    U[k][p] = cs * ukp - sn * ukq;
    U[k][q] = sn * ukp + cs * ukq;
  }
}

__device__ __forceinline__ void dlt_solve(Dlt& s) {
  double a[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      a[r][c] = s.A[0][r] * s.A[0][c] + s.A[1][r] * s.A[1][c] + s.A[2][r] * s.A[2][c] + s.A[3][r] * s.A[3][c];
      s.U[r][c] = r == c ? 1.0 : 0.0;
    }
#pragma unroll 1
  for (int sweep = 0; sweep < JACOBI_SWEEPS; ++sweep) {
    jacobi_rotate<0, 1>(a, s.U);
    jacobi_rotate<0, 2>(a, s.U);
    jacobi_rotate<0, 3>(a, s.U);
    jacobi_rotate<1, 2>(a, s.U);
    jacobi_rotate<1, 3>(a, s.U);
    jacobi_rotate<2, 3>(a, s.U);
  }
  s.imin = 0;
  s.lmin = a[0][0];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    s.lam[i] = a[i][i];
    if (a[i][i] < s.lmin) s.imin = i, s.lmin = a[i][i];
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    double vi = 0.0;
#pragma unroll
    for (int j = 0; j < 4; ++j) vi = j == s.imin ? s.U[i][j] : vi;
    s.v[i] = vi;
  }
  if (s.v[3] < 0.0) {
#pragma unroll
    for (int i = 0; i < 4; ++i) s.v[i] = -s.v[i];
  }
}

// rows x1 E1[2] - E1[0], y1 E1[2] - E1[1], x2 E2[2] - E2[0], y2 E2[2] - E2[1] (kornia triangulate_points)
__device__ __forceinline__ void dlt_rows(Dlt& s, const float* __restrict__ E1, const float* __restrict__ E2, double x1, double y1,
                                         double x2, double y2) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    s.A[0][c] = x1 * (double)E1[8 + c] - (double)E1[c];
    s.A[1][c] = y1 * (double)E1[8 + c] - (double)E1[4 + c];
    s.A[2][c] = x2 * (double)E2[8 + c] - (double)E2[c];
    s.A[3][c] = y2 * (double)E2[8 + c] - (double)E2[4 + c];
  }
}

// gradient of X = v[:3] * homog_scale(v[3]) wrt the two image points of the pair: rows (2 * role, 2 * role + 1) of A,
// role 0 = first camera of the pair, 1 = second.  g_A = (A v) w^T + (A w) v^T with w = -(M - lam I)^+ g_v.
__device__ __forceinline__ void dlt_point_grad(const Dlt& s, const float* __restrict__ E, int role, const double gX[3], double& gx,
                                               double& gy) {
  const double z = s.v[3];
  const double sc = homog_scale(z);
  double gv[4] = {gX[0] * sc, gX[1] * sc, gX[2] * sc, 0.0};
  if (fabs(z) > HOMOG_EPS) gv[3] = -sc * sc * (gX[0] * s.v[0] + gX[1] * s.v[1] + gX[2] * s.v[2]);
  double w[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const double gap = s.lam[i] - s.lmin;
    if (i == s.imin || !(gap > 0.0)) continue;
    const double coef = -(s.U[0][i] * gv[0] + s.U[1][i] * gv[1] + s.U[2][i] * gv[2] + s.U[3][i] * gv[3]) / gap;
#pragma unroll
    for (int r = 0; r < 4; ++r) w[r] += coef * s.U[r][i];
  }
  double ew = 0.0, ev = 0.0;  // E[2, :] . w, E[2, :] . v
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    ew += (double)E[8 + c] * w[c];
    ev += (double)E[8 + c] * s.v[c];
  }
  double av[2], aw[2];
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int r = 2 * role + rr;
    av[rr] = s.A[r][0] * s.v[0] + s.A[r][1] * s.v[1] + s.A[r][2] * s.v[2] + s.A[r][3] * s.v[3];
    aw[rr] = s.A[r][0] * w[0] + s.A[r][1] * w[1] + s.A[r][2] * w[2] + s.A[r][3] * w[3];
  }
  gx = av[0] * ew + aw[0] * ev;
  gy = av[1] * ew + aw[1] * ev;
}

__device__ __forceinline__ int pair_index(int i, int j, int V) { return i * V - i * (i + 1) / 2 + (j - i - 1); }

// ---- projection: K E (4x4) -> two dehomogenisations -> optional distortion -> optional frame -> model ---------------
struct Proj {
  double c[3];   // K E [X; 1], after the first dehomogenisation
  double s1, s2;  // the two homog_scale factors
  double u, v;   // pinhole projection (pixels)
  double x, y;   // normalised coordinates fed to the distortion (when applied)
};

__device__ __forceinline__ void project(const float* __restrict__ K, const float* __restrict__ E, const double X[3], Proj& p) {
  double cam[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) cam[r] = (double)E[4 * r] * X[0] + (double)E[4 * r + 1] * X[1] + (double)E[4 * r + 2] * X[2] + (double)E[4 * r + 3];
  p.s1 = homog_scale(1.0);  // the homogeneous row of K4 E4 is (0, 0, 0, 1)
#pragma unroll
  for (int r = 0; r < 3; ++r) p.c[r] = ((double)K[3 * r] * cam[0] + (double)K[3 * r + 1] * cam[1] + (double)K[3 * r + 2] * cam[2]) * p.s1;
  p.s2 = homog_scale(p.c[2]);
  p.u = p.c[0] * p.s2;
  p.v = p.c[1] * p.s2;
}

__device__ __forceinline__ void distort(const Pinhole& c, const Dist& d, Proj& p, double& ud, double& vd) {
  const double x = (p.u - c.cx) / c.fx, y = (p.v - c.cy) / c.fy;
  p.x = x;
  p.y = y;
  const double r2 = x * x + y * y;
  const double rad = (1.0 + d.k1 * r2 + d.k2 * r2 * r2 + d.k3 * r2 * r2 * r2) / (1.0 + d.k4 * r2 + d.k5 * r2 * r2 + d.k6 * r2 * r2 * r2);
  const double xd = x * rad + 2.0 * d.p1 * x * y + d.p2 * (r2 + 2.0 * x * x) + d.s1 * r2 + d.s2 * r2 * r2;
  const double yd = y * rad + d.p1 * (r2 + 2.0 * y * y) + 2.0 * d.p2 * x * y + d.s3 * r2 + d.s4 * r2 * r2;
  ud = c.fx * xd + c.cx;
  vd = c.fy * yd + c.cy;
}

// (gud, gvd) on the distorted pixel -> gradient on the undistorted pixel (p.x, p.y recorded by distort)
__device__ __forceinline__ void distort_adj(const Pinhole& c, const Dist& d, const Proj& p, double gud, double gvd, double& gu, double& gv) {
  const double x = p.x, y = p.y, r2 = x * x + y * y;
  const double N = 1.0 + d.k1 * r2 + d.k2 * r2 * r2 + d.k3 * r2 * r2 * r2, dN = d.k1 + 2.0 * d.k2 * r2 + 3.0 * d.k3 * r2 * r2;
  const double D = 1.0 + d.k4 * r2 + d.k5 * r2 * r2 + d.k6 * r2 * r2 * r2, dD = d.k4 + 2.0 * d.k5 * r2 + 3.0 * d.k6 * r2 * r2;
  const double rad = N / D, drad = (dN * D - N * dD) / (D * D);
  const double ts = d.s1 + 2.0 * d.s2 * r2, tt = d.s3 + 2.0 * d.s4 * r2;
  const double xd_x = rad + 2.0 * x * x * drad + 2.0 * d.p1 * y + 6.0 * d.p2 * x + 2.0 * x * ts;
  const double xd_y = 2.0 * x * y * drad + 2.0 * d.p1 * x + 2.0 * d.p2 * y + 2.0 * y * ts;
  const double yd_x = 2.0 * x * y * drad + 2.0 * d.p1 * x + 2.0 * d.p2 * y + 2.0 * x * tt;
  const double yd_y = rad + 2.0 * y * y * drad + 6.0 * d.p1 * y + 2.0 * d.p2 * x + 2.0 * y * tt;
  const double gxd = gud * c.fx, gyd = gvd * c.fy;
  gu = (gxd * xd_x + gyd * yd_x) / c.fx;
  gv = (gxd * xd_y + gyd * yd_y) / c.fy;
}

// (gu, gv) on the pinhole projection -> gradient on X
__device__ __forceinline__ void project_adj(const float* __restrict__ K, const float* __restrict__ E, const Proj& p, double gu, double gv,
                                            double gX[3]) {
  double gc[3] = {gu * p.s2, gv * p.s2, 0.0};
  if (fabs(p.c[2]) > HOMOG_EPS) gc[2] = -(gu * p.c[0] + gv * p.c[1]) * p.s2 * p.s2;
  double gcam[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) gcam[j] = ((double)K[j] * gc[0] + (double)K[3 + j] * gc[1] + (double)K[6 + j] * gc[2]) * p.s1;
#pragma unroll
  for (int j = 0; j < 3; ++j) gX[j] += (double)E[j] * gcam[0] + (double)E[4 + j] * gcam[1] + (double)E[8 + j] * gcam[2];
}

// frame_to_model (bboxes.py:150-169): bbox = [x, y, h, w] of this view; `grad` drops the offset (its linear part)
__device__ __forceinline__ void frame_to_model(const float* __restrict__ bb, float model_h, float model_w, bool grad, double& x, double& y) {
  const double bx = grad ? 0.0 : (double)bb[0], by = grad ? 0.0 : (double)bb[1];
  x = (x - bx) / (double)bb[3] * (double)model_w;
  y = (y - by) / (double)bb[2] * (double)model_h;
}

// the 3-D point of (b, k): points3d[b, k] or, with n_pairs > 0, the NaN-propagating mean over the pair axis
__device__ __forceinline__ bool load_point3d(const float* __restrict__ p3, int n_pairs, int b, int k, int K, double X[3]) {
  if (n_pairs == 0) {
    const float* q = p3 + ((size_t)b * K + k) * 3;
    X[0] = q[0], X[1] = q[1], X[2] = q[2];
  } else {
    X[0] = X[1] = X[2] = 0.0;
    for (int p = 0; p < n_pairs; ++p) {
      const float* q = p3 + (((size_t)b * n_pairs + p) * K + k) * 3;
      X[0] += q[0], X[1] += q[1], X[2] += q[2];
    }
    X[0] /= n_pairs, X[1] /= n_pairs, X[2] /= n_pairs;
  }
  return !(isnan(X[0]) || isnan(X[1]) || isnan(X[2]));
}

// ---- kernels ----------------------------------------------------------------------------------------------------------
// one thread per (b, pair, k): undistort both views, DLT, dehomogenise
__global__ void __launch_bounds__(CAM_THREADS) triangulate_fwd_kernel(const float* __restrict__ pts, const float* __restrict__ Km,
                                                                      const float* __restrict__ Em, const float* __restrict__ dist,
                                                                      int B, int V, int K, int P, float* __restrict__ out) {
  const int n_pairs = V * (V - 1) / 2;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= (int64_t)B * n_pairs * K) return;
  const int k = (int)(tid % K);
  const int pr = (int)((tid / K) % n_pairs);
  const int b = (int)(tid / ((int64_t)K * n_pairs));
  int i = 0, rem = pr;
  while (rem >= V - 1 - i) rem -= V - 1 - i++;
  const int j = i + 1 + rem;
  const int bi = b * V + i, bj = b * V + j;
  double x1, y1, x2, y2;
  undistort(load_pinhole(Km + 9 * bi), load_dist(dist + (size_t)P * bi, P), pts[((size_t)bi * K + k) * 2], pts[((size_t)bi * K + k) * 2 + 1], x1, y1);
  undistort(load_pinhole(Km + 9 * bj), load_dist(dist + (size_t)P * bj, P), pts[((size_t)bj * K + k) * 2], pts[((size_t)bj * K + k) * 2 + 1], x2, y2);
  float* o = out + tid * 3;
  if (isnan(x1) || isnan(y1) || isnan(x2) || isnan(y2)) {
    o[0] = o[1] = o[2] = __int_as_float(0x7fc00000);
    return;
  }
  Dlt s;
  dlt_rows(s, Em + 12 * bi, Em + 12 * bj, x1, y1, x2, y2);
  dlt_solve(s);
  const double sc = homog_scale(s.v[3]);
  o[0] = (float)(s.v[0] * sc);
  o[1] = (float)(s.v[1] * sc);
  o[2] = (float)(s.v[2] * sc);
}

// one thread per (b, view, k): the view's point gradient summed over the pairs that contain the view, other view ascending
__global__ void __launch_bounds__(CAM_THREADS) triangulate_bwd_kernel(const float* __restrict__ pts, const float* __restrict__ Km,
                                                                      const float* __restrict__ Em, const float* __restrict__ dist,
                                                                      const float* __restrict__ gout, int B, int V, int K, int P,
                                                                      float* __restrict__ gpts) {
  const int n_pairs = V * (V - 1) / 2;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= (int64_t)B * V * K) return;
  const int k = (int)(tid % K);
  const int v = (int)((tid / K) % V);
  const int b = (int)(tid / ((int64_t)K * V));
  const int bv = b * V + v;
  const Pinhole cv = load_pinhole(Km + 9 * bv);
  const Dist dv = load_dist(dist + (size_t)P * bv, P);
  double xs[UNDISTORT_ITERS], ys[UNDISTORT_ITERS], x, y;
  undistort(cv, dv, pts[tid * 2], pts[tid * 2 + 1], x, y, xs, ys);
  float* g = gpts + tid * 2;
  if (isnan(x) || isnan(y)) {
    g[0] = g[1] = 0.f;
    return;
  }
  double gx = 0.0, gy = 0.0;
  for (int o = 0; o < V; ++o) {
    if (o == v) continue;
    const int bo = b * V + o;
    double xo, yo;
    undistort(load_pinhole(Km + 9 * bo), load_dist(dist + (size_t)P * bo, P), pts[((size_t)bo * K + k) * 2], pts[((size_t)bo * K + k) * 2 + 1], xo, yo);
    if (isnan(xo) || isnan(yo)) continue;
    const int i = min(v, o), j = max(v, o);
    const float* go = gout + (((size_t)b * n_pairs + pair_index(i, j, V)) * K + k) * 3;
    const double gX[3] = {go[0], go[1], go[2]};
    Dlt s;
    if (v < o)
      dlt_rows(s, Em + 12 * bv, Em + 12 * bo, x, y, xo, yo);
    else
      dlt_rows(s, Em + 12 * bo, Em + 12 * bv, xo, yo, x, y);
    dlt_solve(s);
    double px, py;
    dlt_point_grad(s, Em + 12 * bv, v < o ? 0 : 1, gX, px, py);
    gx += px;
    gy += py;
  }
  double gu, gv;
  undistort_adj(cv, dv, xs, ys, gx, gy, gu, gv);
  g[0] = (float)gu;
  g[1] = (float)gv;
}

// one thread per (b, view, k)
__global__ void __launch_bounds__(CAM_THREADS) project_fwd_kernel(const float* __restrict__ p3, int n_pairs, const float* __restrict__ Km,
                                                                  const float* __restrict__ Em, const float* __restrict__ dist,
                                                                  const float* __restrict__ bbox, float model_h, float model_w, int B,
                                                                  int V, int K, int P, float* __restrict__ out) {
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= (int64_t)B * V * K) return;
  const int k = (int)(tid % K);
  const int v = (int)((tid / K) % V);
  const int b = (int)(tid / ((int64_t)K * V));
  const int bv = b * V + v;
  float* o = out + tid * 2;
  double X[3];
  if (!load_point3d(p3, n_pairs, b, k, K, X)) {
    o[0] = o[1] = __int_as_float(0x7fc00000);
    return;
  }
  Proj p;
  project(Km + 9 * bv, Em + 12 * bv, X, p);
  double u = p.u, w = p.v;
  const Dist d = load_dist(dist + (size_t)P * bv, P);
  if (d.any) distort(load_pinhole(Km + 9 * bv), d, p, u, w);
  if (bbox) frame_to_model(bbox + (size_t)b * 4 * V + 4 * v, model_h, model_w, false, u, w);
  o[0] = (float)u;
  o[1] = (float)w;
}

// one thread per (b, k): gradient summed over the views in order, then spread over the pairs of the mean (1 / n_pairs)
__global__ void __launch_bounds__(CAM_THREADS) project_bwd_kernel(const float* __restrict__ p3, int n_pairs, const float* __restrict__ Km,
                                                                  const float* __restrict__ Em, const float* __restrict__ dist,
                                                                  const float* __restrict__ bbox, float model_h, float model_w,
                                                                  const float* __restrict__ gout, int B, int V, int K, int P,
                                                                  float* __restrict__ gp3) {
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= (int64_t)B * K) return;
  const int k = (int)(tid % K);
  const int b = (int)(tid / K);
  double X[3], gX[3] = {0.0, 0.0, 0.0};
  if (load_point3d(p3, n_pairs, b, k, K, X)) {
    for (int v = 0; v < V; ++v) {
      const int bv = b * V + v;
      const float* go = gout + (((size_t)b * V + v) * K + k) * 2;
      double gu = go[0], gv = go[1];
      if (bbox) frame_to_model(bbox + (size_t)b * 4 * V + 4 * v, model_h, model_w, true, gu, gv);
      Proj p;
      project(Km + 9 * bv, Em + 12 * bv, X, p);
      const Dist d = load_dist(dist + (size_t)P * bv, P);
      if (d.any) {
        double ud, vd;
        const Pinhole c = load_pinhole(Km + 9 * bv);
        distort(c, d, p, ud, vd);
        distort_adj(c, d, p, gu, gv, gu, gv);
      }
      project_adj(Km + 9 * bv, Em + 12 * bv, p, gu, gv, gX);
    }
  }
  if (n_pairs == 0) {
    float* g = gp3 + tid * 3;
    g[0] = (float)gX[0], g[1] = (float)gX[1], g[2] = (float)gX[2];
    return;
  }
  for (int q = 0; q < n_pairs; ++q) {
    float* g = gp3 + (((size_t)b * n_pairs + q) * K + k) * 3;
    g[0] = (float)(gX[0] / n_pairs), g[1] = (float)(gX[1] / n_pairs), g[2] = (float)(gX[2] / n_pairs);
  }
}

__global__ void __launch_bounds__(CAM_THREADS) frame_to_model_kernel(const float* __restrict__ in, int B, int V, int K,
                                                                     const float* __restrict__ bbox, float model_h, float model_w, int grad,
                                                                     float* __restrict__ out) {
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= (int64_t)B * V * K) return;
  const int v = (int)((tid / K) % V);
  const int b = (int)(tid / ((int64_t)K * V));
  double x = in[tid * 2], y = in[tid * 2 + 1];
  frame_to_model(bbox + (size_t)b * 4 * V + 4 * v, model_h, model_w, grad != 0, x, y);
  out[tid * 2] = (float)x;
  out[tid * 2 + 1] = (float)y;
}

// ---- pairwise-projection loss: mean L2 distance over entries with neither side NaN (0 when none) -----------------------
constexpr int PPL_THREADS = 256;

__device__ __forceinline__ bool ppl_entry(const float* __restrict__ targ, const float* __restrict__ pred, int64_t e, int n_pairs, int K,
                                          double diff[3], double& dist) {
  const int k = (int)(e % K);
  const int64_t b = e / ((int64_t)K * n_pairs);
  const float* t = targ + (b * K + k) * 3;
  const float* p = pred + e * 3;
  bool ok = true;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    ok &= !(isnan(t[c]) || isnan(p[c]));
    diff[c] = (double)p[c] - (double)t[c];
  }
  dist = ok ? sqrt(diff[0] * diff[0] + diff[1] * diff[1] + diff[2] * diff[2]) : 0.0;
  return ok;
}

__device__ __forceinline__ double block_sum_d(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double t = 0.0;
#pragma unroll
  for (int w = 0; w < PPL_THREADS / 32; ++w) t += red[w];
  return t;
}

// one CTA; out[0] = loss, out[1] = number of kept entries
__global__ void __launch_bounds__(PPL_THREADS) ppl_fwd_kernel(const float* __restrict__ targ, const float* __restrict__ pred, int64_t n,
                                                              int n_pairs, int K, float* __restrict__ out) {
  __shared__ double red[PPL_THREADS / 32];
  double acc = 0.0, cnt = 0.0;
  for (int64_t e = threadIdx.x; e < n; e += PPL_THREADS) {
    double diff[3], d;
    if (ppl_entry(targ, pred, e, n_pairs, K, diff, d)) {
      acc += d;
      cnt += 1.0;
    }
  }
  acc = block_sum_d(acc, red);
  cnt = block_sum_d(cnt, red);
  if (threadIdx.x == 0) {
    out[0] = cnt > 0.0 ? (float)(acc / cnt) : 0.f;
    out[1] = (float)cnt;
  }
}

__global__ void __launch_bounds__(CAM_THREADS) ppl_bwd_kernel(const float* __restrict__ targ, const float* __restrict__ pred, int64_t n,
                                                              int n_pairs, int K, const float* __restrict__ fwd_out,
                                                              const float* __restrict__ gout, float* __restrict__ gpred) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  double diff[3], d;
  const bool ok = ppl_entry(targ, pred, e, n_pairs, K, diff, d);
  const double cnt = fwd_out[1];
  const double s = (ok && d > 0.0 && cnt > 0.0) ? (double)gout[0] / cnt / d : 0.0;
#pragma unroll
  for (int c = 0; c < 3; ++c) gpred[e * 3 + c] = s != 0.0 ? (float)(diff[c] * s) : 0.f;  // dropped entries: diff may be NaN
}

inline unsigned n_blocks(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

}  // namespace
}  // namespace lpb

#define CAM_CHECK_SHAPE(name, V, K, P, min_views)                                                                              \
  LPB_REQUIRE(B >= 0 && K >= 1 && V >= (min_views) && V <= lpb::CAM_MAX_VIEWS, name ": bad V (%d) or K (%d)", V, K);            \
  LPB_REQUIRE(P == 4 || P == 5 || P == 8 || P == 12, name ": bad P (%d): distortion needs 4, 5, 8 or 12 coefficients", P)

extern "C" int lpb_triangulate_pairs_fwd(const float* points, const float* intrinsics, const float* extrinsics, const float* dist,
                                         int B, int V, int K, int P, float* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(points && intrinsics && extrinsics && dist && out, "triangulate_pairs_fwd: null pointer");
  CAM_CHECK_SHAPE("triangulate_pairs_fwd", V, K, P, 2);
  const int64_t n = (int64_t)B * (V * (V - 1) / 2) * K;
  if (n == 0) return LPB_OK;
  triangulate_fwd_kernel<<<n_blocks(n, CAM_THREADS), CAM_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(points, intrinsics, extrinsics,
                                                                                                           dist, B, V, K, P, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_triangulate_pairs_bwd(const float* points, const float* intrinsics, const float* extrinsics, const float* dist,
                                         const float* grad_out, int B, int V, int K, int P, float* grad_points, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(points && intrinsics && extrinsics && dist && grad_out && grad_points, "triangulate_pairs_bwd: null pointer");
  CAM_CHECK_SHAPE("triangulate_pairs_bwd", V, K, P, 2);
  const int64_t n = (int64_t)B * V * K;
  if (n == 0) return LPB_OK;
  triangulate_bwd_kernel<<<n_blocks(n, CAM_THREADS), CAM_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      points, intrinsics, extrinsics, dist, grad_out, B, V, K, P, grad_points);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_project_points_fwd(const float* points3d, int n_pairs, const float* intrinsics, const float* extrinsics,
                                      const float* dist, const float* bbox, float model_height, float model_width, int B, int V,
                                      int K, int P, float* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(points3d && intrinsics && extrinsics && dist && out, "project_points_fwd: null pointer");
  CAM_CHECK_SHAPE("project_points_fwd", V, K, P, 1);
  LPB_REQUIRE(n_pairs >= 0 && (!bbox || (model_height > 0.f && model_width > 0.f)), "project_points_fwd: bad n_pairs or model size");
  const int64_t n = (int64_t)B * V * K;
  if (n == 0) return LPB_OK;
  project_fwd_kernel<<<n_blocks(n, CAM_THREADS), CAM_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      points3d, n_pairs, intrinsics, extrinsics, dist, bbox, model_height, model_width, B, V, K, P, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_project_points_bwd(const float* points3d, int n_pairs, const float* intrinsics, const float* extrinsics,
                                      const float* dist, const float* bbox, float model_height, float model_width,
                                      const float* grad_out, int B, int V, int K, int P, float* grad_points3d, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(points3d && intrinsics && extrinsics && dist && grad_out && grad_points3d, "project_points_bwd: null pointer");
  CAM_CHECK_SHAPE("project_points_bwd", V, K, P, 1);
  LPB_REQUIRE(n_pairs >= 0 && (!bbox || (model_height > 0.f && model_width > 0.f)), "project_points_bwd: bad n_pairs or model size");
  const int64_t n = (int64_t)B * K;
  if (n == 0) return LPB_OK;
  project_bwd_kernel<<<n_blocks(n, CAM_THREADS), CAM_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(
      points3d, n_pairs, intrinsics, extrinsics, dist, bbox, model_height, model_width, grad_out, B, V, K, P, grad_points3d);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_frame_to_model(const float* keypoints, int B, int V, int K, const float* bbox, float model_height, float model_width,
                                  int grad, float* out, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(keypoints && bbox && out, "frame_to_model: null pointer");
  LPB_REQUIRE(B >= 0 && V >= 1 && K >= 1 && model_height > 0.f && model_width > 0.f, "frame_to_model: bad shape");
  const int64_t n = (int64_t)B * V * K;
  if (n == 0) return LPB_OK;
  frame_to_model_kernel<<<n_blocks(n, CAM_THREADS), CAM_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(keypoints, B, V, K, bbox,
                                                                                                          model_height, model_width, grad, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_pairwise_projections_loss_fwd(const float* targets, const float* preds, int B, int n_pairs, int K, float* out,
                                                 void* stream) {
  using namespace lpb;
  LPB_REQUIRE(targets && preds && out, "pairwise_projections_loss_fwd: null pointer");
  LPB_REQUIRE(B >= 0 && n_pairs >= 1 && K >= 1, "pairwise_projections_loss_fwd: bad shape");
  ppl_fwd_kernel<<<1, PPL_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(targets, preds, (int64_t)B * n_pairs * K, n_pairs, K, out);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}

extern "C" int lpb_pairwise_projections_loss_bwd(const float* targets, const float* preds, int B, int n_pairs, int K, const float* fwd_out,
                                                 const float* grad_out, float* grad_preds, void* stream) {
  using namespace lpb;
  LPB_REQUIRE(targets && preds && fwd_out && grad_out && grad_preds, "pairwise_projections_loss_bwd: null pointer");
  LPB_REQUIRE(B >= 0 && n_pairs >= 1 && K >= 1, "pairwise_projections_loss_bwd: bad shape");
  const int64_t n = (int64_t)B * n_pairs * K;
  if (n == 0) return LPB_OK;
  ppl_bwd_kernel<<<n_blocks(n, CAM_THREADS), CAM_THREADS, 0, static_cast<cudaStream_t>(stream)>>>(targets, preds, n, n_pairs, K, fwd_out,
                                                                                                   grad_out, grad_preds);
  LPB_CUDA(cudaGetLastError());
  return LPB_OK;
}
