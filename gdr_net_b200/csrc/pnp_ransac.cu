// Test-time RANSAC-PnP of the evaluator on the device (SURVEY.md 8f row f-4; reference core/gdrn_modeling/gdrn_evaluator.py:316-436
// `process_pnp_ransac`: per instance, on the host, `get_img_model_points_with_coords2d` :89-126 + `misc.pnp_v2`
// lib/pysixd/misc.py:145-194 = cv2.solvePnPRansac(flags=SOLVEPNP_EPNP, reprojectionError=3, iterationsCount=100)).
//
// The arithmetic is OpenCV's (third-party, not under /root/reference); oracle/pnp_oracle.py restates it and is pinned against
// the installed cv2 (EPnP: 1e-14; RANSAC: identical inlier sets).  This file follows that restatement:
//
//   gather    one CTA per ROI: model points (xyz - 0.5) * extent and image points coord2d * (W, H) in fp32 like the reference,
//             selection mask > thr & |xyz_c| > 1e-4 extent_c, compacted IN ROW-MAJOR ORDER (the RANSAC subsets index this order)
//   hypothesis one CTA per (RANSAC iteration, ROI): cv::RNG((uint64)-1) replayed up to this iteration -> 5 distinct indices ->
//             EPnP on the 5 points -> squared reprojection error of all points (float, <= thr^2) -> inlier count.  OpenCV runs
//             the iterations one after the other and shortens the loop from the inlier ratio; the subsets do not depend on the
//             results, so all iterations are evaluated at once and the sequential bookkeeping is replayed afterwards.
//   final     one CTA per ROI: replay of `count > max(best, 4)` / RANSACUpdateNumIters over the iteration results, inlier mask
//             of the winning model, EPnP over all inliers (the sums over points are block reductions), pose out.
//
// EPnP (Lepetit, Moreno-Noguer, Fua, IJCV 2009) as OpenCV runs it: control points = centroid + sqrt(lambda_i / n) u_i from the
// PCA of the model points -- the SIGN of u_i matters at the 1e-4 level for noisy data, so the 3x3 / 12x12 / 6xk decompositions
// are the same one-sided Jacobi SVD OpenCV uses (rotation order, V accumulated from the identity, selection sort); barycentric
// coordinates; M^T M (12x12) accumulated as sum_i (a a^T) (x) S_i; its 4 smallest singular vectors; L (6x10), rho; three beta
// initialisations, 5 Gauss-Newton steps each; R, t by absolute orientation; the candidate with the smallest reprojection error.
// All of it in fp64.  n == 5 points: EPnP over all points (OpenCV's npoints == model_points shortcut); n < 5: ok = 0.
#include <math.h>

#include "gdrn_internal.h"

namespace gdrn {
namespace {

// CTA sizes are compile-time parameters; every loop below strides by them (tests/emu builds this file for the host with one
// thread per CTA to single-step the algorithm against cv2 without a GPU -- test infrastructure, never part of the library).
#ifndef GDRN_PNP_THREADS
#define GDRN_PNP_THREADS 128
#endif
#ifndef GDRN_PNP_HYP_THREADS
#define GDRN_PNP_HYP_THREADS 32  // one warp per RANSAC hypothesis: the EPnP of 5 points is serial work, more CTAs per SM win
#endif
#ifndef GDRN_PNP_GATHER_THREADS
#define GDRN_PNP_GATHER_THREADS 1024
#endif
#ifndef GDRN_LAUNCH
#define GDRN_LAUNCH(kernel, grid, block, stream, ...) kernel<<<grid, block, 0, stream>>>(__VA_ARGS__)
#endif
constexpr int kPnpThreads = GDRN_PNP_THREADS;
constexpr int kPnpWarps = (kPnpThreads + 31) / 32;
constexpr int kHypThreads = GDRN_PNP_HYP_THREADS;
constexpr int kHypWarps = (kHypThreads + 31) / 32;
static_assert(kHypThreads <= kPnpThreads, "EpnpShared::red is sized for the larger CTA");
constexpr int kGatherThreads = GDRN_PNP_GATHER_THREADS;
constexpr int kGatherWarps = (kGatherThreads + 31) / 32;

struct Cam {
    double fu, fv, uc, vc;
};

// ------------------------------------------------------------------------------------------------ serial linear algebra
// One-sided Jacobi SVD on the n rows (length m, stride lda) of At, i.e. on the columns of A.  On return the rows are the LEFT
// singular vectors (normalised), W the singular values (descending), the rows of Vt the right singular vectors.
__device__ void jacobi_svd(double* At, int lda, double* W, double* Vt, int ldv, int m, int n) {
    const double eps = 2.220446049250313e-16 * 10;
    for (int i = 0; i < n; ++i) {
        double sd = 0;
        for (int k = 0; k < m; ++k) sd += At[i * lda + k] * At[i * lda + k];
        W[i] = sd;
        if (Vt) {
            for (int k = 0; k < n; ++k) Vt[i * ldv + k] = 0;
            Vt[i * ldv + i] = 1;
        }
    }
    const int max_iter = m > 30 ? m : 30;
    for (int iter = 0; iter < max_iter; ++iter) {
        bool changed = false;
        for (int i = 0; i < n - 1; ++i)
            for (int j = i + 1; j < n; ++j) {
                double* Ai = At + i * lda;
                double* Aj = At + j * lda;
                double a = W[i], p = 0, b = W[j];
                for (int k = 0; k < m; ++k) p += Ai[k] * Aj[k];
                if (fabs(p) <= eps * sqrt(a * b)) continue;
                p *= 2;
                const double beta = a - b, gamma = hypot(p, beta);
                double c, s;
                if (beta < 0) {
                    const double delta = (gamma - beta) * 0.5;
                    s = sqrt(delta / gamma);
                    c = p / (gamma * s * 2);
                } else {
                    c = sqrt((gamma + beta) / (gamma * 2));
                    s = p / (gamma * c * 2);
                }
                a = b = 0;
                for (int k = 0; k < m; ++k) {
                    const double t0 = c * Ai[k] + s * Aj[k];
                    const double t1 = -s * Ai[k] + c * Aj[k];
                    Ai[k] = t0;
                    Aj[k] = t1;
                    a += t0 * t0;
                    b += t1 * t1;
                }
                W[i] = a;
                W[j] = b;
                changed = true;
                if (Vt) {
                    double* Vi = Vt + i * ldv;
                    double* Vj = Vt + j * ldv;
                    for (int k = 0; k < n; ++k) {
                        const double t0 = c * Vi[k] + s * Vj[k];
                        const double t1 = -s * Vi[k] + c * Vj[k];
                        Vi[k] = t0;
                        Vj[k] = t1;
                    }
                }
            }
        if (!changed) break;
    }
    for (int i = 0; i < n; ++i) {
        double sd = 0;
        for (int k = 0; k < m; ++k) sd += At[i * lda + k] * At[i * lda + k];
        W[i] = sqrt(sd);
    }
    for (int i = 0; i < n - 1; ++i) {
        int j = i;
        for (int k = i + 1; k < n; ++k)
            if (W[j] < W[k]) j = k;
        if (i != j) {
            double t = W[i];
            W[i] = W[j];
            W[j] = t;
            for (int k = 0; k < m; ++k) {
                t = At[i * lda + k];
                At[i * lda + k] = At[j * lda + k];
                At[j * lda + k] = t;
            }
            if (Vt)
                for (int k = 0; k < n; ++k) {
                    t = Vt[i * ldv + k];
                    Vt[i * ldv + k] = Vt[j * ldv + k];
                    Vt[j * ldv + k] = t;
                }
        }
    }
    for (int i = 0; i < n; ++i) {
        const double s = W[i] > 2.2250738585072014e-308 ? 1.0 / W[i] : 0.0;
        for (int k = 0; k < m; ++k) At[i * lda + k] *= s;
    }
}

// min-norm least squares  min |A x - b|,  A [6][nc] row-major, through the SVD with OpenCV's back-substitution threshold
__device__ void svd_lstsq6(const double* A, int nc, const double* b, double* x) {
    double At[5 * 6], W[5], Vt[5 * 5];
    for (int j = 0; j < nc; ++j)
        for (int i = 0; i < 6; ++i) At[j * 6 + i] = A[i * nc + j];
    jacobi_svd(At, 6, W, Vt, 5, 6, nc);
    double thr = 0;
    for (int j = 0; j < nc; ++j) thr += W[j];
    thr *= 2.220446049250313e-16 * 2;
    for (int k = 0; k < nc; ++k) x[k] = 0;
    for (int j = 0; j < nc; ++j) {
        if (fabs(W[j]) <= thr) continue;
        double ub = 0;
        for (int i = 0; i < 6; ++i) ub += At[j * 6 + i] * b[i];
        ub /= W[j];
        for (int k = 0; k < nc; ++k) x[k] += ub * Vt[j * 5 + k];
    }
}

// Householder QR least squares for the 6 x 4 Gauss-Newton systems (A, b are overwritten); returns false when A is singular
__device__ bool qr_lstsq64(double* A, double* b, double* x) {
    constexpr int nr = 6, nc = 4;
    double diag[nc];
    for (int k = 0; k < nc; ++k) {
        double norm = 0;
        for (int i = k; i < nr; ++i) norm += A[i * nc + k] * A[i * nc + k];
        norm = sqrt(norm);
        if (norm == 0) return false;
        const double alpha = A[k * nc + k] > 0 ? -norm : norm;
        // v = column - alpha e_k, stored in place (v_k in A[k][k]); R_kk = alpha
        A[k * nc + k] -= alpha;
        double vtv = 0;
        for (int i = k; i < nr; ++i) vtv += A[i * nc + k] * A[i * nc + k];
        if (vtv == 0) return false;
        for (int j = k + 1; j < nc; ++j) {
            double dot = 0;
            for (int i = k; i < nr; ++i) dot += A[i * nc + k] * A[i * nc + j];
            const double tau = 2 * dot / vtv;
            for (int i = k; i < nr; ++i) A[i * nc + j] -= tau * A[i * nc + k];
        }
        double dot = 0;
        for (int i = k; i < nr; ++i) dot += A[i * nc + k] * b[i];
        const double tau = 2 * dot / vtv;
        for (int i = k; i < nr; ++i) b[i] -= tau * A[i * nc + k];
        diag[k] = alpha;
    }
    for (int i = nc - 1; i >= 0; --i) {
        double sum = b[i];
        for (int j = i + 1; j < nc; ++j) sum -= A[i * nc + j] * x[j];
        x[i] = sum / diag[i];
    }
    return true;
}

__device__ bool invert3(const double* m, double* inv) {
    const double c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
    const double det = m[0] * c00 + m[1] * c01 + m[2] * c02;
    if (det == 0) {
        for (int i = 0; i < 9; ++i) inv[i] = 0;
        return false;
    }
    const double id = 1.0 / det;
    inv[0] = c00 * id;
    inv[1] = (m[2] * m[7] - m[1] * m[8]) * id;
    inv[2] = (m[1] * m[5] - m[2] * m[4]) * id;
    inv[3] = c01 * id;
    inv[4] = (m[0] * m[8] - m[2] * m[6]) * id;
    inv[5] = (m[2] * m[3] - m[0] * m[5]) * id;
    inv[6] = c02 * id;
    inv[7] = (m[1] * m[6] - m[0] * m[7]) * id;
    inv[8] = (m[0] * m[4] - m[1] * m[3]) * id;
    return true;
}

// ------------------------------------------------------------------------------------------------ block-cooperative EPnP
struct EpnpShared {
    double red[kPnpWarps][40];
    double sums[40];
    double cws[4][3];
    double cinv[9];
    double mtm[144];  // becomes Ut (rows = singular vectors of M^T M, descending singular values)
    double w12[12];
    double L[60];
    double rho[6];
    double betas[3][4];
    double ccs[4][3];
    double pw0[3], pc0[3];
    double R[9], t[3];
    double bestR[9], bestt[3];
    double best_err;
    double sign;
    int first;
    int n_sel;
};

template <int NT, int K>
__device__ void block_sum(double (&v)[K], EpnpShared& S) {
    constexpr int NW = (NT + 31) / 32;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        double x = v[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        if (lane == 0) S.red[warp][k] = x;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += NT) {
        double x = 0;
        for (int w2 = 0; w2 < NW; ++w2) x += S.red[w2][k];
        S.sums[k] = x;
    }
    __syncthreads();
}

__device__ __forceinline__ void alphas_of(const EpnpShared& S, const double* pw, double* a) {
    const double dx = pw[0] - S.cws[0][0], dy = pw[1] - S.cws[0][1], dz = pw[2] - S.cws[0][2];
    a[1] = S.cinv[0] * dx + S.cinv[1] * dy + S.cinv[2] * dz;
    a[2] = S.cinv[3] * dx + S.cinv[4] * dy + S.cinv[5] * dz;
    a[3] = S.cinv[6] * dx + S.cinv[7] * dy + S.cinv[8] * dz;
    a[0] = 1.0 - a[1] - a[2] - a[3];
}

// thread 0: everything between M^T M and the three beta vectors
__device__ void epnp_betas_serial(EpnpShared& S) {
    jacobi_svd(S.mtm, 12, S.w12, nullptr, 0, 12, 12);  // symmetric: rows of A == columns of A
    const double* ut = S.mtm;
    const double* v[4] = {ut + 12 * 11, ut + 12 * 10, ut + 12 * 9, ut + 12 * 8};
    double dv[4][6][3];
    for (int i = 0; i < 4; ++i) {
        int a = 0, b = 1;
        for (int k = 0; k < 6; ++k) {
            for (int c = 0; c < 3; ++c) dv[i][k][c] = v[i][3 * a + c] - v[i][3 * b + c];
            if (++b > 3) {
                ++a;
                b = a + 1;
            }
        }
    }
    auto d = [&](int i, int j, int k) { return dv[i][k][0] * dv[j][k][0] + dv[i][k][1] * dv[j][k][1] + dv[i][k][2] * dv[j][k][2]; };
    for (int k = 0; k < 6; ++k) {
        double* l = S.L + 10 * k;
        l[0] = d(0, 0, k);
        l[1] = 2 * d(0, 1, k);
        l[2] = d(1, 1, k);
        l[3] = 2 * d(0, 2, k);
        l[4] = 2 * d(1, 2, k);
        l[5] = d(2, 2, k);
        l[6] = 2 * d(0, 3, k);
        l[7] = 2 * d(1, 3, k);
        l[8] = 2 * d(2, 3, k);
        l[9] = d(3, 3, k);
    }
    {
        int a = 0, b = 1;
        for (int k = 0; k < 6; ++k) {
            double s = 0;
            for (int c = 0; c < 3; ++c) s += (S.cws[a][c] - S.cws[b][c]) * (S.cws[a][c] - S.cws[b][c]);
            S.rho[k] = s;
            if (++b > 3) {
                ++a;
                b = a + 1;
            }
        }
    }
    double sub[6 * 5], x[5];
    // approximation 1: [B11 B12 B13 B14]
    {
        const int cols[4] = {0, 1, 3, 6};
        for (int i = 0; i < 6; ++i)
            for (int j = 0; j < 4; ++j) sub[i * 4 + j] = S.L[10 * i + cols[j]];
        svd_lstsq6(sub, 4, S.rho, x);
        double* be = S.betas[0];
        if (x[0] < 0) {
            be[0] = sqrt(-x[0]);
            be[1] = -x[1] / be[0];
            be[2] = -x[2] / be[0];
            be[3] = -x[3] / be[0];
        } else {
            be[0] = sqrt(x[0]);
            be[1] = x[1] / be[0];
            be[2] = x[2] / be[0];
            be[3] = x[3] / be[0];
        }
    }
    // approximation 2: [B11 B12 B22]
    {
        for (int i = 0; i < 6; ++i)
            for (int j = 0; j < 3; ++j) sub[i * 3 + j] = S.L[10 * i + j];
        svd_lstsq6(sub, 3, S.rho, x);
        double* be = S.betas[1];
        if (x[0] < 0) {
            be[0] = sqrt(-x[0]);
            be[1] = x[2] < 0 ? sqrt(-x[2]) : 0.0;
        } else {
            be[0] = sqrt(x[0]);
            be[1] = x[2] > 0 ? sqrt(x[2]) : 0.0;
        }
        if (x[1] < 0) be[0] = -be[0];
        be[2] = 0.0;
        be[3] = 0.0;
    }
    // approximation 3: [B11 B12 B22 B13 B23]
    {
        for (int i = 0; i < 6; ++i)
            for (int j = 0; j < 5; ++j) sub[i * 5 + j] = S.L[10 * i + j];
        svd_lstsq6(sub, 5, S.rho, x);
        double* be = S.betas[2];
        if (x[0] < 0) {
            be[0] = sqrt(-x[0]);
            be[1] = x[2] < 0 ? sqrt(-x[2]) : 0.0;
        } else {
            be[0] = sqrt(x[0]);
            be[1] = x[2] > 0 ? sqrt(x[2]) : 0.0;
        }
        if (x[1] < 0) be[0] = -be[0];
        be[2] = x[3] / be[0];
        be[3] = 0.0;
    }
    // Gauss-Newton, 5 steps each
    for (int c = 0; c < 3; ++c) {
        double* b = S.betas[c];
        for (int it = 0; it < 5; ++it) {
            double A[24], r[6], dx[4];
            for (int i = 0; i < 6; ++i) {
                const double* l = S.L + 10 * i;
                A[i * 4 + 0] = 2 * l[0] * b[0] + l[1] * b[1] + l[3] * b[2] + l[6] * b[3];
                A[i * 4 + 1] = l[1] * b[0] + 2 * l[2] * b[1] + l[4] * b[2] + l[7] * b[3];
                A[i * 4 + 2] = l[3] * b[0] + l[4] * b[1] + 2 * l[5] * b[2] + l[8] * b[3];
                A[i * 4 + 3] = l[6] * b[0] + l[7] * b[1] + l[8] * b[2] + 2 * l[9] * b[3];
                r[i] = S.rho[i] - (l[0] * b[0] * b[0] + l[1] * b[0] * b[1] + l[2] * b[1] * b[1] + l[3] * b[0] * b[2] + l[4] * b[1] * b[2] +
                                   l[5] * b[2] * b[2] + l[6] * b[0] * b[3] + l[7] * b[1] * b[3] + l[8] * b[2] * b[3] + l[9] * b[3] * b[3]);
            }
            if (!qr_lstsq64(A, r, dx)) break;
            for (int k = 0; k < 4; ++k) b[k] += dx[k];
        }
    }
}

// Points come through a functor `pt(i, pw, uv) -> bool` (i in [0, n_total): false = not part of the set).  All threads of the
// CTA call this; the result is in S.bestR / S.bestt (valid for every thread after the call).
template <int NT, class PointFn>
__device__ void epnp_block(const PointFn& pt, int n_total, const Cam cam, EpnpShared& S) {
    const int tid = threadIdx.x;
    if (tid == 0) {
        S.first = 0x7fffffff;
        S.best_err = INFINITY;
        for (int i = 0; i < 9; ++i) S.bestR[i] = (i % 4 == 0) ? 1.0 : 0.0;
        S.bestt[0] = S.bestt[1] = S.bestt[2] = 0.0;
    }
    __syncthreads();
    // centroid
    {
        double v[4] = {0, 0, 0, 0};
        int first = 0x7fffffff;
        for (int i = tid; i < n_total; i += NT) {
            double pw[3], uv[2];
            if (!pt(i, pw, uv)) continue;
            v[0] += pw[0];
            v[1] += pw[1];
            v[2] += pw[2];
            v[3] += 1.0;
            if (i < first) first = i;
        }
        if (first != 0x7fffffff) atomicMin(&S.first, first);
        block_sum<NT, 4>(v, S);
        if (tid == 0) {
            S.n_sel = (int)S.sums[3];
            for (int c = 0; c < 3; ++c) S.cws[0][c] = S.pw0[c] = S.sums[c] / S.sums[3];
        }
        __syncthreads();
    }
    const int n = S.n_sel;
    if (n < 4) return;
    // PCA of the model points -> control points, inverse of [c1-c0 c2-c0 c3-c0]
    {
        double v[6] = {0, 0, 0, 0, 0, 0};
        for (int i = tid; i < n_total; i += NT) {
            double pw[3], uv[2];
            if (!pt(i, pw, uv)) continue;
            const double x = pw[0] - S.cws[0][0], y = pw[1] - S.cws[0][1], z = pw[2] - S.cws[0][2];
            v[0] += x * x;
            v[1] += x * y;
            v[2] += x * z;
            v[3] += y * y;
            v[4] += y * z;
            v[5] += z * z;
        }
        block_sum<NT, 6>(v, S);
        if (tid == 0) {
            double C[9] = {S.sums[0], S.sums[1], S.sums[2], S.sums[1], S.sums[3], S.sums[4], S.sums[2], S.sums[4], S.sums[5]};
            double dc[3];
            jacobi_svd(C, 3, dc, nullptr, 0, 3, 3);
            for (int i = 1; i < 4; ++i) {
                const double k = sqrt(dc[i - 1] / n);
                for (int c = 0; c < 3; ++c) S.cws[i][c] = S.cws[0][c] + k * C[3 * (i - 1) + c];
            }
            double cc[9];
            for (int r = 0; r < 3; ++r)
                for (int j = 0; j < 3; ++j) cc[3 * r + j] = S.cws[j + 1][r] - S.cws[0][r];
            invert3(cc, S.cinv);
        }
        __syncthreads();
    }
    // M^T M = sum_i (a a^T) (x) S_i,  S_i = [[fu^2, 0, fu du], [0, fv^2, fv dv], [fu du, fv dv, du^2 + dv^2]]
    {
        double v[40];
#pragma unroll
        for (int k = 0; k < 40; ++k) v[k] = 0;
        for (int i = tid; i < n_total; i += NT) {
            double pw[3], uv[2], a[4];
            if (!pt(i, pw, uv)) continue;
            alphas_of(S, pw, a);
            const double du = cam.uc - uv[0], dvv = cam.vc - uv[1], q = du * du + dvv * dvv;
            int e = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int k = j; k < 4; ++k) {
                    const double aa = a[j] * a[k];
                    v[e] += aa;
                    v[e + 1] += aa * du;
                    v[e + 2] += aa * dvv;
                    v[e + 3] += aa * q;
                    e += 4;
                }
        }
        block_sum<NT, 40>(v, S);
        for (int e16 = tid; e16 < 16; e16 += NT) {
            const int j = e16 >> 2, k = e16 & 3;
            const int lo = j < k ? j : k, hi = j < k ? k : j;
            // index of pair (lo, hi), lo <= hi, in the order (0,0) (0,1) (0,2) (0,3) (1,1) ...
            const int e = 4 * (lo * 4 - lo * (lo - 1) / 2 + (hi - lo));
            const double aa = S.sums[e], adu = S.sums[e + 1], adv = S.sums[e + 2], aq = S.sums[e + 3];
            double* m = S.mtm + (3 * j) * 12 + 3 * k;
            m[0] = cam.fu * cam.fu * aa;
            m[1] = 0;
            m[2] = cam.fu * adu;
            m[12] = 0;
            m[13] = cam.fv * cam.fv * aa;
            m[14] = cam.fv * adv;
            m[24] = cam.fu * adu;
            m[25] = cam.fv * adv;
            m[26] = aq;
        }
        __syncthreads();
    }
    if (tid == 0) epnp_betas_serial(S);
    __syncthreads();
    // three candidates: R, t by absolute orientation between camera-frame and model points, reprojection error
    for (int c = 0; c < 3; ++c) {
        if (tid == 0) {
            for (int j = 0; j < 4; ++j)
                for (int k = 0; k < 3; ++k) {
                    double s = 0;
                    for (int i = 0; i < 4; ++i) s += S.betas[c][i] * S.mtm[12 * (11 - i) + 3 * j + k];
                    S.ccs[j][k] = s;
                }
            // sign: the FIRST point of the set must be in front of the camera
            double pw[3], uv[2], a[4];
            pt(S.first, pw, uv);
            alphas_of(S, pw, a);
            const double z = a[0] * S.ccs[0][2] + a[1] * S.ccs[1][2] + a[2] * S.ccs[2][2] + a[3] * S.ccs[3][2];
            if (z < 0.0)
                for (int j = 0; j < 4; ++j)
                    for (int k = 0; k < 3; ++k) S.ccs[j][k] = -S.ccs[j][k];
        }
        __syncthreads();
        {
            double v[3] = {0, 0, 0};
            for (int i = tid; i < n_total; i += NT) {
                double pw[3], uv[2], a[4];
                if (!pt(i, pw, uv)) continue;
                alphas_of(S, pw, a);
                for (int k = 0; k < 3; ++k) v[k] += a[0] * S.ccs[0][k] + a[1] * S.ccs[1][k] + a[2] * S.ccs[2][k] + a[3] * S.ccs[3][k];
            }
            block_sum<NT, 3>(v, S);
            for (int k = tid; k < 3; k += NT) S.pc0[k] = S.sums[k] / n;
            __syncthreads();
        }
        {
            double v[9];
#pragma unroll
            for (int k = 0; k < 9; ++k) v[k] = 0;
            for (int i = tid; i < n_total; i += NT) {
                double pw[3], uv[2], a[4], pc[3];
                if (!pt(i, pw, uv)) continue;
                alphas_of(S, pw, a);
                for (int k = 0; k < 3; ++k)
                    pc[k] = a[0] * S.ccs[0][k] + a[1] * S.ccs[1][k] + a[2] * S.ccs[2][k] + a[3] * S.ccs[3][k] - S.pc0[k];
#pragma unroll
                for (int j = 0; j < 3; ++j)
#pragma unroll
                    for (int k = 0; k < 3; ++k) v[3 * j + k] += pc[j] * (pw[k] - S.pw0[k]);
            }
            block_sum<NT, 9>(v, S);
            if (tid == 0) {
                // SVD of ABt (rows of `at` = columns of ABt): ABt = U diag(w) V^T,  R = U V^T
                double at[9], w[3], vt[9];
                for (int j = 0; j < 3; ++j)
                    for (int k = 0; k < 3; ++k) at[3 * k + j] = S.sums[3 * j + k];
                jacobi_svd(at, 3, w, vt, 3, 3, 3);  // rows of `at` are now the u_i
                for (int i = 0; i < 3; ++i)
                    for (int j = 0; j < 3; ++j) S.R[3 * i + j] = at[0 + i] * vt[0 + j] + at[3 + i] * vt[3 + j] + at[6 + i] * vt[6 + j];
                const double det = S.R[0] * (S.R[4] * S.R[8] - S.R[5] * S.R[7]) - S.R[1] * (S.R[3] * S.R[8] - S.R[5] * S.R[6]) +
                                   S.R[2] * (S.R[3] * S.R[7] - S.R[4] * S.R[6]);
                if (det < 0) {
                    S.R[6] = -S.R[6];
                    S.R[7] = -S.R[7];
                    S.R[8] = -S.R[8];
                }
                for (int i = 0; i < 3; ++i)
                    S.t[i] = S.pc0[i] - (S.R[3 * i] * S.pw0[0] + S.R[3 * i + 1] * S.pw0[1] + S.R[3 * i + 2] * S.pw0[2]);
            }
            __syncthreads();
        }
        {
            double v[1] = {0};
            for (int i = tid; i < n_total; i += NT) {
                double pw[3], uv[2];
                if (!pt(i, pw, uv)) continue;
                const double X = S.R[0] * pw[0] + S.R[1] * pw[1] + S.R[2] * pw[2] + S.t[0];
                const double Y = S.R[3] * pw[0] + S.R[4] * pw[1] + S.R[5] * pw[2] + S.t[1];
                const double iz = 1.0 / (S.R[6] * pw[0] + S.R[7] * pw[1] + S.R[8] * pw[2] + S.t[2]);
                const double ue = cam.uc + cam.fu * X * iz, ve = cam.vc + cam.fv * Y * iz;
                v[0] += sqrt((uv[0] - ue) * (uv[0] - ue) + (uv[1] - ve) * (uv[1] - ve));
            }
            block_sum<NT, 1>(v, S);
            if (tid == 0) {
                const double err = S.sums[0] / n;
                if (c == 0 || err < S.best_err) {  // N = 1; if (e2 < e1) N = 2; if (e3 < e_N) N = 3
                    S.best_err = err;
                    for (int i = 0; i < 9; ++i) S.bestR[i] = S.R[i];
                    for (int i = 0; i < 3; ++i) S.bestt[i] = S.t[i];
                }
            }
            __syncthreads();
        }
    }
}

// ------------------------------------------------------------------------------------------------ kernels
// Per-ROI scratch layout (doubles): pts [HW][5] = (X, Y, Z, u, v)
__global__ void __launch_bounds__(kGatherThreads) pnp_gather_kernel(const float* __restrict__ mask, const float* __restrict__ xyz,
                                                                    const float* __restrict__ coord2d, const float* __restrict__ extents,
                                                                    const float* __restrict__ im_wh, int HW, int mask_mode, float mask_thr,
                                                                    double* __restrict__ pts, int* __restrict__ counts) {
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    __shared__ float s_min[kGatherWarps], s_max[kGatherWarps];
    __shared__ int s_warp[kGatherWarps];
    __shared__ int s_base;
    const float* m = mask + (long)b * HW * (mask_mode == 3 ? 2 : 1);  // mode 3: two mask planes per ROI
    float mn = INFINITY, mx = -INFINITY;
    if (mask_mode == 1) {  // L1 mask head: per-ROI min-max normalisation (engine_utils.py:113-118)
        for (int i = tid; i < HW; i += kGatherThreads) {
            mn = fminf(mn, m[i]);
            mx = fmaxf(mx, m[i]);
        }
        for (int o = 16; o > 0; o >>= 1) {
            mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
        if (lane == 0) {
            s_min[warp] = mn;
            s_max[warp] = mx;
        }
        __syncthreads();
        mn = s_min[0];
        mx = s_max[0];
        for (int w2 = 1; w2 < kGatherWarps; ++w2) {
            mn = fminf(mn, s_min[w2]);
            mx = fmaxf(mx, s_max[w2]);
        }
    }
    if (tid == 0) s_base = 0;
    __syncthreads();
    const float ex = extents[b * 3], ey = extents[b * 3 + 1], ez = extents[b * 3 + 2];
    const float iw = im_wh[b * 2], ih = im_wh[b * 2 + 1];
    const float tx = __fmul_rn(0.0001f, ex), ty = __fmul_rn(0.0001f, ey), tz = __fmul_rn(0.0001f, ez);
    double* out = pts + (long)b * HW * 5;
    for (int base = 0; base < HW; base += kGatherThreads) {  // row-major order is preserved chunk by chunk
        const int i = base + tid;
        bool sel = false;
        float X = 0, Y = 0, Z = 0, u = 0, v = 0;
        if (i < HW) {
            float mv = m[i];
            if (mask_mode == 1) mv = __fdiv_rn(__fsub_rn(mv, mn), __fsub_rn(mx, mn));
            else if (mask_mode == 2) mv = 1.f / (1.f + expf(-mv));
            else if (mask_mode == 3) mv = m[HW + i] > mv ? 1.f : 0.f;  // CE head: argmax over 2 channels, a tie is class 0
            X = __fmul_rn(__fsub_rn(xyz[((long)b * 3 + 0) * HW + i], 0.5f), ex);
            Y = __fmul_rn(__fsub_rn(xyz[((long)b * 3 + 1) * HW + i], 0.5f), ey);
            Z = __fmul_rn(__fsub_rn(xyz[((long)b * 3 + 2) * HW + i], 0.5f), ez);
            u = __fmul_rn(coord2d[((long)b * 2 + 0) * HW + i], iw);
            v = __fmul_rn(coord2d[((long)b * 2 + 1) * HW + i], ih);
            sel = mv > mask_thr && fabsf(X) > tx && fabsf(Y) > ty && fabsf(Z) > tz;
        }
        const unsigned bal = __ballot_sync(0xffffffffu, sel);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        int off = s_base;
        for (int w2 = 0; w2 < warp; ++w2) off += s_warp[w2];
        off += __popc(bal & ((1u << lane) - 1u));
        if (sel) {
            double* o = out + (long)off * 5;
            o[0] = X;
            o[1] = Y;
            o[2] = Z;
            o[3] = u;
            o[4] = v;
        }
        __syncthreads();
        if (tid == 0) {
            int tot = 0;
            for (int w2 = 0; w2 < kGatherWarps; ++w2) tot += s_warp[w2];
            s_base += tot;
        }
        __syncthreads();
    }
    if (tid == 0) counts[b] = s_base;
}

struct CvRng {  // cv::RNG: multiply-with-carry
    unsigned long long state;
    __device__ unsigned next() {
        state = (unsigned long long)(unsigned)state * 4164903690ull + (unsigned)(state >> 32);
        return (unsigned)state;
    }
    __device__ int uniform(int a, int b) { return a == b ? a : (int)(next() % (unsigned)(b - a) + a); }
};

__device__ __forceinline__ bool is_inlier(const double* R, const double* t, const Cam& cam, const double* p, double thr2) {
    const double X = R[0] * p[0] + R[1] * p[1] + R[2] * p[2] + t[0];
    const double Y = R[3] * p[0] + R[4] * p[1] + R[5] * p[2] + t[1];
    double z = R[6] * p[0] + R[7] * p[1] + R[8] * p[2] + t[2];
    z = z != 0.0 ? 1.0 / z : 1.0;
    const double du = p[3] - (X * z * cam.fu + cam.uc), dv = p[4] - (Y * z * cam.fv + cam.vc);
    const float err = (float)(du * du + dv * dv);
    return (double)err <= thr2;
}

__device__ __forceinline__ Cam load_cam(const float* K, int b) {
    Cam c;
    c.fu = (double)K[b * 9 + 0];
    c.fv = (double)K[b * 9 + 4];
    c.uc = (double)K[b * 9 + 2];
    c.vc = (double)K[b * 9 + 5];
    return c;
}

// solvePnP maps the image points to normalised coordinates (undistortPoints, zero distortion) and EPnP maps them back
__device__ __forceinline__ void epnp_uv(const Cam& cam, const double* p, double* uv) {
    uv[0] = (p[3] - cam.uc) * (1.0 / cam.fu) * cam.fu + cam.uc;
    uv[1] = (p[4] - cam.vc) * (1.0 / cam.fv) * cam.fv + cam.vc;
}

__global__ void __launch_bounds__(kHypThreads) pnp_hypothesis_kernel(const double* __restrict__ pts, const int* __restrict__ counts,
                                                                    const float* __restrict__ K, int HW, int iters, double thr2,
                                                                    double* __restrict__ models, int* __restrict__ hyp_counts) {
    const int it = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int n = counts[b];
    __shared__ EpnpShared S;
    __shared__ double sub[5][5];
    __shared__ int s_cnt[kHypWarps];
    if (n <= 5) {  // n == 5: direct solve in the final kernel; n < 5: no pose
        if (tid == 0) hyp_counts[b * iters + it] = 0;
        return;
    }
    const double* P = pts + (long)b * HW * 5;
    const Cam cam = load_cam(K, b);
    if (tid == 0) {
        CvRng rng{0xffffffffffffffffull};
        int idx[5];
        for (int k = 0; k <= it; ++k)
            for (int i = 0; i < 5; ++i) {
                int c;
                bool dup;
                do {
                    c = rng.uniform(0, n);
                    dup = false;
                    for (int j = 0; j < i; ++j) dup |= idx[j] == c;
                } while (dup);
                idx[i] = c;
            }
        for (int i = 0; i < 5; ++i)
            for (int k = 0; k < 5; ++k) sub[i][k] = P[(long)idx[i] * 5 + k];
    }
    __syncthreads();
    auto pt = [&](int i, double* pw, double* uv) {
        pw[0] = sub[i][0];
        pw[1] = sub[i][1];
        pw[2] = sub[i][2];
        epnp_uv(cam, sub[i], uv);
        return true;
    };
    epnp_block<kHypThreads>(pt, 5, cam, S);
    __syncthreads();
    double R[9], t[3];
    for (int i = 0; i < 9; ++i) R[i] = S.bestR[i];
    for (int i = 0; i < 3; ++i) t[i] = S.bestt[i];
    int cnt = 0;
    for (int i = tid; i < n; i += kHypThreads) cnt += is_inlier(R, t, cam, P + (long)i * 5, thr2) ? 1 : 0;
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((tid & 31) == 0) s_cnt[tid >> 5] = cnt;
    __syncthreads();
    if (tid == 0) {
        int tot = 0;
        for (int w2 = 0; w2 < kHypWarps; ++w2) tot += s_cnt[w2];
        hyp_counts[b * iters + it] = tot;
        double* m = models + ((long)b * iters + it) * 12;
        for (int i = 0; i < 9; ++i) m[i] = R[i];
        for (int i = 0; i < 3; ++i) m[9 + i] = t[i];
    }
}

// RANSACUpdateNumIters (OpenCV calib3d ptsetreg.cpp)
__device__ int ransac_update_num_iters(double p, double ep, int model_points, int max_iters) {
    p = fmin(fmax(p, 0.0), 1.0);
    ep = fmin(fmax(ep, 0.0), 1.0);
    double num = fmax(1.0 - p, 2.2250738585072014e-308);
    double denom = 1.0 - pow(1.0 - ep, (double)model_points);
    if (denom < 2.2250738585072014e-308) return 0;
    num = log(num);
    denom = log(denom);
    return (denom >= 0 || -num >= max_iters * (-denom)) ? max_iters : (int)rint(num / denom);
}

__global__ void __launch_bounds__(kPnpThreads) pnp_final_kernel(const double* __restrict__ pts, const int* __restrict__ counts,
                                                               const float* __restrict__ K, const double* __restrict__ models,
                                                               const int* __restrict__ hyp_counts, int HW, int iters, double thr2,
                                                               double confidence, unsigned char* __restrict__ flags,
                                                               float* __restrict__ out_pose, int* __restrict__ out_info) {
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = counts[b];
    __shared__ EpnpShared S;
    __shared__ int s_best, s_iters_run;
    __shared__ int s_cnt[kPnpWarps];
    const double* P = pts + (long)b * HW * 5;
    unsigned char* F = flags + (long)b * HW;
    const Cam cam = load_cam(K, b);
    if (tid == 0) {
        int best = -1, best_count = 0, niters = iters, it = 0;
        if (n > 5) {
            for (; it < niters; ++it) {
                const int c = hyp_counts[b * iters + it];
                if (c > (best_count > 4 ? best_count : 4)) {
                    best_count = c;
                    best = it;
                    niters = ransac_update_num_iters(confidence, (double)(n - c) / n, 5, niters);
                }
            }
        }
        s_best = best;
        s_iters_run = it;
    }
    __syncthreads();
    const int best = s_best;
    int n_in = 0;
    if (n == 5) {
        for (int i = tid; i < n; i += kPnpThreads) F[i] = 1;
        n_in = 5;
    } else if (best >= 0) {
        double R[9], t[3];
        const double* m = models + ((long)b * iters + best) * 12;
        for (int i = 0; i < 9; ++i) R[i] = m[i];
        for (int i = 0; i < 3; ++i) t[i] = m[9 + i];
        int cnt = 0;
        for (int i = tid; i < n; i += kPnpThreads) {
            const bool in = is_inlier(R, t, cam, P + (long)i * 5, thr2);
            F[i] = in ? 1 : 0;
            cnt += in ? 1 : 0;
        }
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        if ((tid & 31) == 0) s_cnt[tid >> 5] = cnt;
        __syncthreads();
        for (int w2 = 0; w2 < kPnpWarps; ++w2) n_in += s_cnt[w2];
    }
    __syncthreads();  // flags visible to the whole CTA
    const bool ok = n_in >= 5;
    if (ok) {
        auto pt = [&](int i, double* pw, double* uv) {
            if (!F[i]) return false;
            const double* p = P + (long)i * 5;
            pw[0] = p[0];
            pw[1] = p[1];
            pw[2] = p[2];
            epnp_uv(cam, p, uv);
            return true;
        };
        epnp_block<kPnpThreads>(pt, n, cam, S);
        __syncthreads();
    }
    for (int e = tid; e < 12; e += kPnpThreads) {
        float v;
        if (ok) {
            const int r = e >> 2, c = e & 3;
            v = (float)(c < 3 ? S.bestR[3 * r + c] : S.bestt[r]);
        } else {
            v = (e == 0 || e == 5 || e == 10) ? 1.f : 0.f;  // rvec = tvec = 0 -> identity, like the untouched outputs of a failed call
        }
        out_pose[b * 12 + e] = v;
    }
    if (tid == 0) {
        out_info[b * 4 + 0] = n;
        out_info[b * 4 + 1] = n_in;
        out_info[b * 4 + 2] = s_iters_run;
        out_info[b * 4 + 3] = ok ? 1 : 0;
    }
}

// ------------------------------------------------------------------------------------------------ network-initialised iterative PnP
// cv2.solvePnP(SOLVEPNP_ITERATIVE, useExtrinsicGuess=True) of the evaluator's net_iter_pnp mode (gdrn_evaluator.py:187-314):
// OpenCV's cvFindExtrinsicCameraParams2 with a guess = Levenberg-Marquardt (CvLevMarq) on p = (rvec, tvec), residual = projected
// pixel - image point.  oracle/net_pnp_oracle.py restates it (pinned against cv2: 1e-9) and this kernel follows that restatement:
//   CALC_J    J, r at p -> JtJ, Jtr (one block reduction of 28 sums); prev = p; p = prev - solve(JtJ, diag * (1 + 10^l), Jtr)
//             by SVD; the first time prevErr = |r|
//   CHECK_ERR err = |r(p)|; err > prevErr and ++l <= 16: re-solve from prev, check again; else l = max(l - 1, -16), ++iters,
//             stop at iters >= max_iters or |p - prev| / (|prev| + DBL_EPSILON) < FLT_EPSILON, else prevErr = err -> CALC_J
// The serial part (6x6 solve, state machine, Rodrigues both ways) runs on thread 0 with its scratch in shared memory.
struct LmShared {
    double p[6], prev[6];
    double JtJ[36], Jtr[6];
    double At[36], Vt[36], w[6];  // SVD scratch (6x6 solve; the 3x3 re-orthonormalisation uses the leading 9 entries)
    double R[9], dRdr[27];        // R(p[0:3]) and dR / dr (row j = derivative by r_j of the 9 entries of R, row-major)
    double prev_err;
    int lam, iters, phase;  // phase: 0 = check the error again, 1 = new Jacobian, 2 = done
};

// cv::Rodrigues, vector -> matrix, with the 3x9 derivative
__device__ void rodrigues_v2m(const double* r, double* R, double* J) {
    const double theta = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    if (theta < 2.220446049250313e-16) {
        for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0) ? 1.0 : 0.0;
        for (int k = 0; k < 27; ++k) J[k] = 0.0;
        J[5] = -1;
        J[7] = 1;
        J[9 + 2] = 1;
        J[9 + 6] = -1;
        J[18 + 1] = -1;
        J[18 + 3] = 1;
        return;
    }
    const double c = cos(theta), s = sin(theta), c1 = 1.0 - c, itheta = 1.0 / theta;
    const double rx = r[0] * itheta, ry = r[1] * itheta, rz = r[2] * itheta;
    const double rrt[9] = {rx * rx, rx * ry, rx * rz, rx * ry, ry * ry, ry * rz, rx * rz, ry * rz, rz * rz};
    const double r_x[9] = {0, -rz, ry, rz, 0, -rx, -ry, rx, 0};
    const double I[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    for (int k = 0; k < 9; ++k) R[k] = c * I[k] + c1 * rrt[k] + s * r_x[k];
    const double drrt[27] = {rx + rx, ry, rz, ry, 0, 0, rz, 0, 0, 0, rx, 0, rx, ry + ry, rz, 0, rz, 0, 0, 0, rx, 0, 0, ry, rx, ry, rz + rz};
    const double d_r_x[27] = {0, 0, 0, 0, 0, -1, 0, 1, 0, 0, 0, 1, 0, 0, 0, -1, 0, 0, 0, -1, 0, 1, 0, 0, 0, 0, 0};
    for (int i = 0; i < 3; ++i) {
        const double ri = i == 0 ? rx : i == 1 ? ry : rz;
        const double a0 = -s * ri, a1 = (s - 2 * c1 * itheta) * ri, a2 = c1 * itheta, a3 = (c - s * itheta) * ri, a4 = s * itheta;
        for (int k = 0; k < 9; ++k) J[i * 9 + k] = a0 * I[k] + a1 * rrt[k] + a2 * drrt[i * 9 + k] + a3 * r_x[k] + a4 * d_r_x[i * 9 + k];
    }
}

// cv::Rodrigues, matrix -> vector: SVD re-orthonormalisation (R = U V^T), then the axis / angle closed forms with OpenCV's
// theta ~ 0 and theta ~ pi branches.  `at`, `vt`, `w` are 9 / 9 / 3 doubles of scratch.
__device__ void rodrigues_m2v(const double* Rin, double* r, double* at, double* vt, double* w) {
    for (int j = 0; j < 3; ++j)
        for (int k = 0; k < 3; ++k) at[3 * k + j] = Rin[3 * j + k];  // rows of `at` = columns of R
    jacobi_svd(at, 3, w, vt, 3, 3, 3);
    double R[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R[3 * i + j] = at[0 + i] * vt[0 + j] + at[3 + i] * vt[3 + j] + at[6 + i] * vt[6 + j];
    double rx = R[7] - R[5], ry = R[2] - R[6], rz = R[3] - R[1];
    const double s = sqrt((rx * rx + ry * ry + rz * rz) * 0.25);
    double c = (R[0] + R[4] + R[8] - 1) * 0.5;
    c = c > 1. ? 1. : c < -1. ? -1. : c;
    double theta = acos(c);
    if (s < 1e-5) {
        if (c > 0) {
            rx = ry = rz = 0;
        } else {
            rx = sqrt(fmax((R[0] + 1) * 0.5, 0.));
            ry = sqrt(fmax((R[4] + 1) * 0.5, 0.)) * (R[1] < 0 ? -1. : 1.);
            rz = sqrt(fmax((R[8] + 1) * 0.5, 0.)) * (R[2] < 0 ? -1. : 1.);
            if (fabs(rx) < fabs(ry) && fabs(rx) < fabs(rz) && (R[5] > 0) != (ry * rz > 0)) rz = -rz;
            theta /= sqrt(rx * rx + ry * ry + rz * rz);
            rx *= theta;
            ry *= theta;
            rz *= theta;
        }
    } else {
        const double vth = 1 / (2 * s) * theta;
        rx *= vth;
        ry *= vth;
        rz *= vth;
    }
    r[0] = rx;
    r[1] = ry;
    r[2] = rz;
}

// cv::solve(A, b, DECOMP_SVD) for the 6x6 damped normal equations, OpenCV's back-substitution threshold (as svd_lstsq6)
__device__ void svd_solve6(LmShared& L, const double* b, double* x) {
    for (int j = 0; j < 6; ++j)
        for (int i = 0; i < 6; ++i) L.At[j * 6 + i] = L.JtJ[i * 6 + j] * (i == j ? 1.0 + exp(L.lam * log(10.)) : 1.0);
    jacobi_svd(L.At, 6, L.w, L.Vt, 6, 6, 6);
    double thr = 0;
    for (int j = 0; j < 6; ++j) thr += L.w[j];
    thr *= 2.220446049250313e-16 * 2;
    for (int k = 0; k < 6; ++k) x[k] = 0;
    for (int j = 0; j < 6; ++j) {
        if (fabs(L.w[j]) <= thr) continue;
        double ub = 0;
        for (int i = 0; i < 6; ++i) ub += L.At[j * 6 + i] * b[i];
        ub /= L.w[j];
        for (int k = 0; k < 6; ++k) x[k] += ub * L.Vt[j * 6 + k];
    }
}

// CvLevMarq::step: p = prev - solve(JtJ with its diagonal * (1 + 10^lam), Jtr); then R, dR/dr at the new p (thread 0)
__device__ void lm_step(LmShared& L) {
    double x[6];
    svd_solve6(L, L.Jtr, x);
    for (int k = 0; k < 6; ++k) L.p[k] = L.prev[k] - x[k];
    rodrigues_v2m(L.p, L.R, L.dRdr);
}

// Residual of one point (model point q[0:3], image point q[3:5]) at (L.R, L.p[3:6]); with J: its two Jacobian rows
template <bool WANT_J>
__device__ __forceinline__ void lm_point(const LmShared& L, const Cam& cam, const double* q, double& ru, double& rv, double* ju,
                                         double* jv) {
    const double X = q[0], Y = q[1], Z = q[2];
    const double Xc = L.R[0] * X + L.R[1] * Y + L.R[2] * Z + L.p[3];
    const double Yc = L.R[3] * X + L.R[4] * Y + L.R[5] * Z + L.p[4];
    const double Zc = L.R[6] * X + L.R[7] * Y + L.R[8] * Z + L.p[5];
    const double z = Zc != 0.0 ? 1.0 / Zc : 1.0;
    const double x = Xc * z, y = Yc * z;
    ru = cam.fu * x + cam.uc - q[3];
    rv = cam.fv * y + cam.vc - q[4];
    if (WANT_J) {
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const double* d = L.dRdr + 9 * j;
            const double dX = X * d[0] + Y * d[1] + Z * d[2];
            const double dY = X * d[3] + Y * d[4] + Z * d[5];
            const double dZ = X * d[6] + Y * d[7] + Z * d[8];
            ju[j] = cam.fu * (z * (dX - x * dZ));
            jv[j] = cam.fv * (z * (dY - y * dZ));
        }
        ju[3] = cam.fu * z;
        ju[4] = 0.0;
        ju[5] = cam.fu * (-x * z);
        jv[3] = 0.0;
        jv[4] = cam.fv * z;
        jv[5] = cam.fv * (-y * z);
    }
}

// CALC_J: JtJ (21 unique entries), Jtr, |r|^2 over all points in one reduction; thread 0 then takes the damped step
template <int NT>
__device__ void lm_calc_j(const double* P, int n, const Cam& cam, LmShared& L, EpnpShared& S) {
    double v[28];
#pragma unroll
    for (int k = 0; k < 28; ++k) v[k] = 0;
    for (int i = threadIdx.x; i < n; i += NT) {
        // re-read R / dRdr from shared memory per point: hoisted next to the 28 accumulators they spill to local memory
        asm volatile("" ::: "memory");
        double ru, rv, ju[6], jv[6];
        lm_point<true>(L, cam, P + (long)i * 5, ru, rv, ju, jv);
        int e = 0;
#pragma unroll
        for (int a = 0; a < 6; ++a) {
#pragma unroll
            for (int c = a; c < 6; ++c) v[e++] += ju[a] * ju[c] + jv[a] * jv[c];
            v[21 + a] += ju[a] * ru + jv[a] * rv;
        }
        v[27] += ru * ru + rv * rv;
    }
    block_sum<NT, 28>(v, S);
    if (threadIdx.x == 0) {
        int e = 0;
        for (int a = 0; a < 6; ++a) {
            for (int c = a; c < 6; ++c, ++e) L.JtJ[a * 6 + c] = L.JtJ[c * 6 + a] = S.sums[e];
            L.Jtr[a] = S.sums[21 + a];
            L.prev[a] = L.p[a];
        }
        if (L.iters == 0) L.prev_err = sqrt(S.sums[27]);
        lm_step(L);
    }
    __syncthreads();
}

// Per-ROI scratch: the gathered points of pnp_gather_kernel.  R_init [B][3][3], t_init [B][3] = the network pose (float32).
__global__ void __launch_bounds__(kPnpThreads) pnp_lm_kernel(const double* __restrict__ pts, const int* __restrict__ counts,
                                                            const float* __restrict__ K, const float* __restrict__ R_init,
                                                            const float* __restrict__ t_init, int HW, int max_iters,
                                                            float* __restrict__ out_pose, int* __restrict__ out_info) {
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = counts[b];
    __shared__ EpnpShared S;
    __shared__ LmShared L;
    if (n < 4) {  // cv2 refuses fewer than 4 points without a guess; the evaluator keeps the network pose below 4
        for (int e = tid; e < 12; e += kPnpThreads) out_pose[b * 12 + e] = (e & 3) < 3 ? R_init[b * 9 + 3 * (e >> 2) + (e & 3)] : t_init[b * 3 + (e >> 2)];
        if (tid == 0) {
            out_info[b * 4 + 0] = n;
            out_info[b * 4 + 1] = 0;
            out_info[b * 4 + 2] = 0;
            out_info[b * 4 + 3] = 0;
        }
        return;
    }
    const double* P = pts + (long)b * HW * 5;
    const Cam cam = load_cam(K, b);
    if (tid == 0) {
        // rvec0 = cv2.Rodrigues(R_net) on the float32 rotation: computed in double, handed back in float32
        double R0[9], r0[3];
        for (int k = 0; k < 9; ++k) R0[k] = (double)R_init[b * 9 + k];
        rodrigues_m2v(R0, r0, L.At, L.Vt, L.w);
        for (int k = 0; k < 3; ++k) {
            L.p[k] = (double)(float)r0[k];
            L.p[3 + k] = (double)t_init[b * 3 + k];
        }
        rodrigues_v2m(L.p, L.R, L.dRdr);
        L.lam = -3;
        L.iters = 0;
    }
    __syncthreads();
    lm_calc_j<kPnpThreads>(P, n, cam, L, S);
    for (;;) {
        double v[1] = {0};
        for (int i = tid; i < n; i += kPnpThreads) {
            double ru, rv;
            lm_point<false>(L, cam, P + (long)i * 5, ru, rv, nullptr, nullptr);
            v[0] += ru * ru + rv * rv;
        }
        block_sum<kPnpThreads, 1>(v, S);
        if (tid == 0) {
            const double err = sqrt(S.sums[0]);
            L.phase = 0;
            if (!(err > L.prev_err && ++L.lam <= 16)) {
                L.lam = L.lam - 1 > -16 ? L.lam - 1 : -16;
                double dn = 0, pn = 0;
                for (int k = 0; k < 6; ++k) {
                    dn += (L.p[k] - L.prev[k]) * (L.p[k] - L.prev[k]);
                    pn += L.prev[k] * L.prev[k];
                }
                if (++L.iters >= max_iters || sqrt(dn) / (sqrt(pn) + 2.220446049250313e-16) < 1.1920928955078125e-07) {
                    L.phase = 2;
                } else {
                    L.prev_err = err;
                    L.phase = 1;
                }
            } else {
                lm_step(L);  // error went up: more damping, same Jacobian
            }
        }
        __syncthreads();
        const int phase = L.phase;
        if (phase == 2) break;
        if (phase == 1) lm_calc_j<kPnpThreads>(P, n, cam, L, S);
    }
    if (tid == 0) {
        // the evaluator passes float32 guess arrays, into which cv2 writes the solution; R = cv2.Rodrigues(rvec)
        double r[3];
        for (int k = 0; k < 3; ++k) r[k] = (double)(float)L.p[k];
        rodrigues_v2m(r, L.R, L.dRdr);
        for (int e = 0; e < 12; ++e) {
            const int i = e >> 2, c = e & 3;
            out_pose[b * 12 + e] = c < 3 ? (float)L.R[3 * i + c] : (float)L.p[3 + i];
        }
        out_info[b * 4 + 0] = n;
        out_info[b * 4 + 1] = L.iters;
        out_info[b * 4 + 2] = 1;
        out_info[b * 4 + 3] = 0;
    }
}

}  // namespace
}  // namespace gdrn

extern "C" long gdrn_pnp_iterative_workspace_bytes(int B, int HW) {
    size_t n = 0;
    n += (size_t)B * HW * 5 * sizeof(double);  // points
    n += (size_t)B * sizeof(int);              // counts
    return (long)(n + 256);
}

extern "C" int gdrn_pnp_iterative(const float* mask, const float* xyz, const float* coord2d, const float* extents, const float* im_wh,
                                  const float* K, const float* R_init, const float* t_init, int B, int H, int W, int mask_mode,
                                  float mask_thr, int max_iters, void* workspace, long workspace_bytes, float* out_pose, int* out_info,
                                  void* stream_) {
    using namespace gdrn;
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!mask || !xyz || !coord2d || !extents || !im_wh || !K || !R_init || !t_init || !workspace || !out_pose || !out_info)
        return set_error(GDRN_ERR_ARG, "gdrn_pnp_iterative: null pointer");
    if (B <= 0 || H <= 0 || W <= 0 || max_iters <= 0 || max_iters > 1000 || mask_mode < 0 || mask_mode > 3)
        return set_error(GDRN_ERR_ARG, "gdrn_pnp_iterative: bad sizes (B=%d H=%d W=%d max_iters=%d mask_mode=%d)", B, H, W, max_iters,
                         mask_mode);
    const int HW = H * W;
    if (workspace_bytes < gdrn_pnp_iterative_workspace_bytes(B, HW))
        return set_error(GDRN_ERR_ARG, "gdrn_pnp_iterative: workspace too small (%ld < %ld)", workspace_bytes,
                         gdrn_pnp_iterative_workspace_bytes(B, HW));
    if ((reinterpret_cast<uintptr_t>(workspace) & 7) != 0)
        return set_error(GDRN_ERR_ARG, "gdrn_pnp_iterative: workspace must be 8-byte aligned");
    double* pts = (double*)workspace;
    int* counts = (int*)((char*)workspace + (size_t)B * HW * 5 * sizeof(double));
    GDRN_LAUNCH(pnp_gather_kernel, dim3(B), dim3(kGatherThreads), stream, mask, xyz, coord2d, extents, im_wh, HW, mask_mode, mask_thr, pts,
                counts);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    GDRN_LAUNCH(pnp_lm_kernel, dim3(B), dim3(kPnpThreads), stream, pts, counts, K, R_init, t_init, HW, max_iters, out_pose, out_info);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return GDRN_OK;
}

extern "C" long gdrn_pnp_ransac_workspace_bytes(int B, int HW, int iters) {
    size_t n = 0;
    n += (size_t)B * HW * 5 * sizeof(double);     // points
    n += (size_t)B * iters * 12 * sizeof(double);  // models
    n += (size_t)B * sizeof(int);                  // counts
    n += (size_t)B * iters * sizeof(int);          // inlier counts per iteration
    n += (size_t)B * HW;                           // inlier flags
    return (long)(n + 256);
}

extern "C" int gdrn_pnp_ransac(const float* mask, const float* xyz, const float* coord2d, const float* extents, const float* im_wh,
                               const float* K, int B, int H, int W, int mask_mode, float mask_thr, double reproj_err, int iters,
                               double confidence, void* workspace, long workspace_bytes, float* out_pose, int* out_info,
                               unsigned char* out_inliers, void* stream_) {
    using namespace gdrn;
    cudaStream_t stream = (cudaStream_t)stream_;
    if (!mask || !xyz || !coord2d || !extents || !im_wh || !K || !workspace || !out_pose || !out_info)
        return set_error(GDRN_ERR_ARG, "gdrn_pnp_ransac: null pointer");
    if (B <= 0 || H <= 0 || W <= 0 || iters <= 0 || iters > 10000 || mask_mode < 0 || mask_mode > 3)
        return set_error(GDRN_ERR_ARG, "gdrn_pnp_ransac: bad sizes (B=%d H=%d W=%d iters=%d mask_mode=%d)", B, H, W, iters, mask_mode);
    const int HW = H * W;
    if (workspace_bytes < gdrn_pnp_ransac_workspace_bytes(B, HW, iters))
        return set_error(GDRN_ERR_ARG, "gdrn_pnp_ransac: workspace too small (%ld < %ld)", workspace_bytes,
                         gdrn_pnp_ransac_workspace_bytes(B, HW, iters));
    if ((reinterpret_cast<uintptr_t>(workspace) & 7) != 0) return set_error(GDRN_ERR_ARG, "gdrn_pnp_ransac: workspace must be 8-byte aligned");
    char* ws = (char*)workspace;
    double* pts = (double*)ws;
    ws += (size_t)B * HW * 5 * sizeof(double);
    double* models = (double*)ws;
    ws += (size_t)B * iters * 12 * sizeof(double);
    int* counts = (int*)ws;
    ws += (size_t)B * sizeof(int);
    int* hyp_counts = (int*)ws;
    ws += (size_t)B * iters * sizeof(int);
    unsigned char* flags = out_inliers ? out_inliers : (unsigned char*)ws;
    const double thr2 = reproj_err * reproj_err;
    if (out_inliers) GDRN_CUDA_OK(cudaMemsetAsync(out_inliers, 0, (size_t)B * HW, stream));
    GDRN_LAUNCH(pnp_gather_kernel, dim3(B), dim3(kGatherThreads), stream, mask, xyz, coord2d, extents, im_wh, HW, mask_mode, mask_thr, pts,
                counts);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    GDRN_LAUNCH(pnp_hypothesis_kernel, dim3(iters, B), dim3(kHypThreads), stream, pts, counts, K, HW, iters, thr2, models, hyp_counts);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    GDRN_LAUNCH(pnp_final_kernel, dim3(B), dim3(kPnpThreads), stream, pts, counts, K, models, hyp_counts, HW, iters, thr2, confidence,
                flags, out_pose, out_info);
    GDRN_CUDA_OK(cudaGetLastError());
    count_launch();
    return GDRN_OK;
}
