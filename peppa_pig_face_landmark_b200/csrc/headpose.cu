// Head pose from 10 facial landmarks, batched on the GPU (SURVEY 8f-4): replaces the OpenCV calls of
// the reference's Skps/core/headpose/pose.py:48-77 get_head_pose():
//   cv2.solvePnP(object_pts, image_pts, K, 0)  -> (rvec, tvec)     [SOLVEPNP_ITERATIVE: DLT start + Levenberg-Marquardt]
//   cv2.projectPoints(reprojectsrc, ...)       -> 8 cube corners
//   cv2.Rodrigues + cv2.decomposeProjectionMatrix -> Euler angles in degrees
// One warp per face, float64.  The start value follows OpenCV's (direct linear transform on normalised image points,
// rotation = orthogonal polar factor), the refinement minimises the pixel reprojection error over (rvec, tvec) with
// Levenberg-Marquardt until the step is below 1e-12 - i.e. the same local minimum OpenCV's 20-iteration solver approaches;
// agreement with cv2 is checked in tests/test_headpose_gpu.py (tolerance stated there), stationarity and agreement over
// the pose space in tests/test_headpose_edges_gpu.py.  The damping grows until a step improves (up to lambda = 1e16), so
// the solver ends no worse than cv2 on small noisy faces too; a few of those (about 1 in 100 below 50 px) lie in a long
// flat valley that it has not crossed after 100 iterations, where cv2's 20 have not either.
// The lanes share the parallel parts: the 12x12 normal matrix, the row / column updates of every Jacobi rotation, the 12
// residual evaluations of the numeric Jacobian, J^T J / J^T e and the 6x6 elimination.  Every sum runs in a fixed order
// (the one-thread solver's, except the Jacobi stopping test), so a face's pose does not depend on the other faces of a launch.
#include <math.h>

#include "../../include/skps_b200.h"
#include "common.h"
#include "mpipe_kernels.h"

namespace skps {

constexpr int HP_PTS = 10;

__device__ void rodrigues(const double* r, double* R) {
    const double th = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
    if (th < 1e-12) {
        R[0] = 1; R[1] = -r[2]; R[2] = r[1]; R[3] = r[2]; R[4] = 1; R[5] = -r[0]; R[6] = -r[1]; R[7] = r[0]; R[8] = 1;
        return;
    }
    const double kx = r[0] / th, ky = r[1] / th, kz = r[2] / th, c = cos(th), s = sin(th), v = 1 - c;
    R[0] = c + kx * kx * v; R[1] = kx * ky * v - kz * s; R[2] = kx * kz * v + ky * s;
    R[3] = ky * kx * v + kz * s; R[4] = c + ky * ky * v; R[5] = ky * kz * v - kx * s;
    R[6] = kz * kx * v - ky * s; R[7] = kz * ky * v + kx * s; R[8] = c + kz * kz * v;
}

// rotation matrix -> rotation vector (cv2.Rodrigues inverse)
__device__ void rodrigues_inv(const double* R, double* r) {
    const double cx = R[7] - R[5], cy = R[2] - R[6], cz = R[3] - R[1];
    const double s = 0.5 * sqrt(cx * cx + cy * cy + cz * cz);
    double c = 0.5 * (R[0] + R[4] + R[8] - 1.0);
    c = c > 1 ? 1 : (c < -1 ? -1 : c);
    const double th = acos(c);
    if (s < 1e-5) {
        if (c > 0) { r[0] = r[1] = r[2] = 0; return; }
        // theta = pi
        double t0 = sqrt(fmax((R[0] + 1) * 0.5, 0.0)), t1 = sqrt(fmax((R[4] + 1) * 0.5, 0.0)) * (R[1] < 0 ? -1 : 1);
        double t2 = sqrt(fmax((R[8] + 1) * 0.5, 0.0)) * (R[2] < 0 ? -1 : 1);
        if (fabs(t0) < fabs(t1) && fabs(t0) < fabs(t2) && ((R[5] > 0) != (t1 * t2 > 0))) t2 = -t2;
        const double n = th / sqrt(t0 * t0 + t1 * t1 + t2 * t2);
        r[0] = t0 * n; r[1] = t1 * n; r[2] = t2 * n;
        return;
    }
    const double k = th / (2 * s);
    r[0] = cx * k; r[1] = cy * k; r[2] = cz * k;
}

__device__ double det3(const double* M) {
    return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}
__device__ void inv3T(const double* M, double* O) {        // O = (M^-1)^T
    const double d = 1.0 / det3(M);
    O[0] = (M[4] * M[8] - M[5] * M[7]) * d; O[1] = (M[5] * M[6] - M[3] * M[8]) * d; O[2] = (M[3] * M[7] - M[4] * M[6]) * d;
    O[3] = (M[2] * M[7] - M[1] * M[8]) * d; O[4] = (M[0] * M[8] - M[2] * M[6]) * d; O[5] = (M[1] * M[6] - M[0] * M[7]) * d;
    O[6] = (M[1] * M[5] - M[2] * M[4]) * d; O[7] = (M[2] * M[3] - M[0] * M[5]) * d; O[8] = (M[0] * M[4] - M[1] * M[3]) * d;
}

__device__ void project(const double* R, const double* t, const float* X, double f, double cx, double cy, double* uv) {
    const double x = R[0] * X[0] + R[1] * X[1] + R[2] * X[2] + t[0];
    const double y = R[3] * X[0] + R[4] * X[1] + R[5] * X[2] + t[1];
    const double z = R[6] * X[0] + R[7] * X[1] + R[8] * X[2] + t[2];
    uv[0] = f * x / z + cx; uv[1] = f * y / z + cy;
}

// Normalise a Givens pair (c, s) the way cv::RQDecomp3x3 does, 1 / sqrt(c^2 + s^2 + DBL_EPSILON), while that is a rotation
// to within sqrt(DBL_EPSILON / (c^2 + s^2)) <= 1.5e-5 in the angle.  Below |(c, s)| = 1e-3 (only the first pair, at
// |cos yaw| < 1e-3) the epsilon would dominate and leave Qx far from a rotation - the Euler triple would then not compose
// back to R (off by up to 2 within 1e-8 of yaw = +-90 degrees) - so there the pair is normalised exactly, and an all-zero
// pair (yaw exactly +-90) is taken as (1, 0), i.e. pitch 0 and the whole rotation about z in the roll.
__device__ __forceinline__ void givens_unit(double& c, double& s) {
    const double n2 = c * c + s * s, z = 1.0 / sqrt(n2 + (n2 >= 1e-6 ? 2.220446049250313e-16 : 0.0));
    c = n2 > 0 ? c * z : 1.0;
    s = n2 > 0 ? s * z : 0.0;
}

// cv::RQDecomp3x3 on a rotation matrix -> Euler angles in degrees (what cv2.decomposeProjectionMatrix returns for [R|t]).
// This is the classic Givens-rotation RQDecomp3x3.  Where the decomposition is not unique it may pick a different triple
// than a given OpenCV build: at an exact 180-degree pitch (R[2][1] = 0 and R[2][2] < 0, e.g. Ry(pi - 0.1): (180, 5.73, 180)
// here, (0, 174.27, 0) from OpenCV 4.13; also the exact 180-degree rotations about some axes) and near yaw = +-90 degrees
// (gimbal lock, where only pitch - roll or pitch + roll is defined).  The triple always composes back to the same
// R = Rz(roll) Ry(yaw) Rx(pitch); tests/test_headpose_edges_gpu.py pins that.
__device__ void euler_rq(const double* Rin, double* eul) {
    double M[9];
    for (int i = 0; i < 9; ++i) M[i] = Rin[i];
    auto mul = [](const double* A, const double* B, double* C) {
        for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
    };
    double s = M[7], c = M[8];
    givens_unit(c, s);
    double Qx[9] = {1, 0, 0, 0, c, s, 0, -s, c}, R[9];
    mul(M, Qx, R);
    s = -R[6]; c = R[8];
    givens_unit(c, s);
    double Qy[9] = {c, 0, -s, 0, 1, 0, s, 0, c};
    mul(R, Qy, M);
    s = M[3]; c = M[4];
    givens_unit(c, s);
    double Qz[9] = {c, s, 0, -s, c, 0, 0, 0, 1};
    mul(M, Qz, R);
    // decomposition ambiguity: diagonal entries of R (except the last) positive; rotate by 180 degrees where needed
    auto T = [](double* Q) { double t; t = Q[1]; Q[1] = Q[3]; Q[3] = t; t = Q[2]; Q[2] = Q[6]; Q[6] = t; t = Q[5]; Q[5] = Q[7]; Q[7] = t; };
    if (R[0] < 0) {
        if (R[4] < 0) {
            Qz[0] = -Qz[0]; Qz[1] = -Qz[1]; Qz[3] = -Qz[3]; Qz[4] = -Qz[4];
        } else {
            T(Qz);
            Qy[0] = -Qy[0]; Qy[2] = -Qy[2]; Qy[6] = -Qy[6]; Qy[8] = -Qy[8];
        }
    } else if (R[4] < 0) {
        T(Qz); T(Qy);
        Qx[4] = -Qx[4]; Qx[5] = -Qx[5]; Qx[7] = -Qx[7]; Qx[8] = -Qx[8];
    }
    const double deg = 180.0 / 3.14159265358979323846;
    auto ac = [](double v) { return acos(v > 1 ? 1.0 : (v < -1 ? -1.0 : v)); };
    eul[0] = ac(Qx[4]) * (Qx[5] >= 0 ? 1 : -1) * deg;
    eul[1] = ac(Qy[0]) * (Qy[6] >= 0 ? 1 : -1) * deg;
    eul[2] = ac(Qz[0]) * (Qz[1] >= 0 ? 1 : -1) * deg;
}


constexpr int HP_WARPS = 4;             // faces (warps) per block

// one warp's scratch
struct PoseSmem {
    float obj[3 * HP_PTS], cube[24];
    double img[2 * HP_PTS];             // image points (float32 values)
    double rows[2][HP_PTS][12];         // the two DLT rows of every point
    double A[144], V[144];              // normal matrix (diagonalised in place) and its eigenvectors
    double ep[12][2 * HP_PTS];          // residuals at p + h_j e_j (row 2j) and p - h_j e_j (row 2j+1)
    double h[6];
    double J[2 * HP_PTS][6];
    double JtJ[36], Jte[6];
    double Mx[6][7];                    // damped normal equations | right-hand side
    double e[2][2 * HP_PTS];            // residuals at the current and at the trial parameters
};

// Butterfly sum: the two lanes of a pair add the same two values, so every lane ends with the same bits.
__device__ __forceinline__ double warp_sum(double v) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Squared reprojection error at p; lanes 0..9 write the residuals of point `lane` to e, every lane returns the sum.
__device__ double warp_residual(const PoseSmem& S, const double* p, double f, double cx, double cy, double* e, int lane) {
    double R[9];
    rodrigues(p, R);
    if (lane < HP_PTS) {
        double uv[2];
        project(R, p + 3, S.obj + 3 * lane, f, cx, cy, uv);
        e[2 * lane] = uv[0] - S.img[2 * lane]; e[2 * lane + 1] = uv[1] - S.img[2 * lane + 1];
    }
    __syncwarp();
    double s = 0;
    for (int i = 0; i < HP_PTS; ++i) s += e[2 * i] * e[2 * i] + e[2 * i + 1] * e[2 * i + 1];
    return s;
}

__global__ void __launch_bounds__(HP_WARPS * 32) head_pose_warp_kernel(const PoseArgs a) {
    __shared__ PoseSmem smem[HP_WARPS];
    const int lane = threadIdx.x & 31;
    const int face = blockIdx.x * HP_WARPS + (threadIdx.x >> 5);
    if (face >= a.G * a.K) return;                  // whole warps leave together
    const int g = face / a.K;
    if (a.count && face - g * a.K >= a.count[g]) return;
    PoseSmem& S = smem[threadIdx.x >> 5];
    const int H = a.hw ? a.hw[2 * g] : a.H, W = a.hw ? a.hw[2 * g + 1] : a.W;
    const double f = (float)W, cx = (float)(W / 2), cy = (float)(H / 2);
    // ---- inputs: the 10 image points rounded to float32 (np.float32(shape[...]) in pose.py), the model
    if (lane < 2 * HP_PTS) {
        int id = a.idx[0];
#pragma unroll
        for (int q = 1; q < HP_PTS; ++q) if ((lane >> 1) == q) id = a.idx[q];
        const size_t at = ((size_t)face * a.P + id) * 2 + (lane & 1);
        S.img[lane] = a.pts64 ? (double)(float)a.pts64[at] : (double)a.pts32[at];
    }
    if (lane == 0) {
#pragma unroll
        for (int q = 0; q < 3 * HP_PTS; ++q) S.obj[q] = a.obj[q];
#pragma unroll
        for (int q = 0; q < 24; ++q) S.cube[q] = a.cube[q];
    }
    __syncwarp();
    // ---- start value: DLT on normalised image points (OpenCV's non-planar branch), rotation = polar factor
    for (int t = lane; t < HP_PTS * 12; t += 32) {  // row 0: X Y Z 1 0 0 0 0 xX xY xZ x, row 1: 0 0 0 0 X Y Z 1 yX yY yZ y
        const int i = t / 12, c = t - 12 * i, k = c & 3;
        const double v = k == 3 ? 1.0 : (double)S.obj[3 * i + k];
        const double x = -(S.img[2 * i] - cx) / f, y = -(S.img[2 * i + 1] - cy) / f;
        S.rows[0][i][c] = c < 4 ? v : (c < 8 ? 0.0 : x * v);
        S.rows[1][i][c] = c < 4 ? 0.0 : (c < 8 ? v : y * v);
    }
    __syncwarp();
    for (int t = lane; t < 144; t += 32) {
        const int r = t / 12, c = t - 12 * r;
        double s = 0;
        for (int i = 0; i < HP_PTS; ++i) s += S.rows[0][i][r] * S.rows[0][i][c] + S.rows[1][i][r] * S.rows[1][i][c];
        S.A[t] = s;
        S.V[t] = (t % 13 == 0) ? 1.0 : 0.0;
    }
    __syncwarp();
    // smallest eigenvector of A: cyclic Jacobi, lanes 0..11 rotate rows / columns of A, lanes 12..23 columns of V
    for (int sweep = 0; sweep < 30; ++sweep) {
        double off = 0;
        for (int t = lane; t < 144; t += 32) if (t % 12 > t / 12) off += S.A[t] * S.A[t];
        if (warp_sum(off) < 1e-30) break;
        for (int p = 0; p < 12; ++p)
            for (int q = p + 1; q < 12; ++q) {
                const double apq = S.A[p * 12 + q];
                if (fabs(apq) < 1e-300) continue;
                const double th = (S.A[q * 12 + q] - S.A[p * 12 + p]) / (2 * apq);
                const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1));
                const double c = 1 / sqrt(t * t + 1), s = t * c;
                __syncwarp();
                if (lane < 12) {
                    const double akp = S.A[lane * 12 + p], akq = S.A[lane * 12 + q];
                    S.A[lane * 12 + p] = c * akp - s * akq; S.A[lane * 12 + q] = s * akp + c * akq;
                } else if (lane < 24) {
                    const int k = lane - 12;
                    const double vkp = S.V[k * 12 + p], vkq = S.V[k * 12 + q];
                    S.V[k * 12 + p] = c * vkp - s * vkq; S.V[k * 12 + q] = s * vkp + c * vkq;
                }
                __syncwarp();
                if (lane < 12) {
                    const double apk = S.A[p * 12 + lane], aqk = S.A[q * 12 + lane];
                    S.A[p * 12 + lane] = c * apk - s * aqk; S.A[q * 12 + lane] = s * apk + c * aqk;
                }
                __syncwarp();
            }
    }
    int m = 0;
    for (int i = 1; i < 12; ++i) if (S.A[i * 13] < S.A[m * 13]) m = i;
    double RR[9] = {S.V[m], S.V[12 + m], S.V[24 + m], S.V[48 + m], S.V[60 + m], S.V[72 + m], S.V[96 + m], S.V[108 + m],
                    S.V[120 + m]};
    double tt[3] = {S.V[36 + m], S.V[84 + m], S.V[132 + m]};
    if (det3(RR) < 0) { for (int i = 0; i < 9; ++i) RR[i] = -RR[i]; for (int i = 0; i < 3; ++i) tt[i] = -tt[i]; }
    double sc = 0;
    for (int i = 0; i < 9; ++i) sc += RR[i] * RR[i];
    sc = sqrt(sc);
    double R[9];
    for (int i = 0; i < 9; ++i) R[i] = RR[i] / (sc / sqrt(3.0));
    for (int it = 0; it < 40; ++it) {                      // Newton iteration to the orthogonal polar factor U V^T
        double iT[9];
        inv3T(R, iT);
        double d = 0;
        for (int i = 0; i < 9; ++i) { const double v = 0.5 * (R[i] + iT[i]); d += fabs(v - R[i]); R[i] = v; }
        if (d < 1e-15) break;
    }
    double p[6];
    rodrigues_inv(R, p);
    for (int i = 0; i < 3; ++i) p[3 + i] = tt[i] * (sqrt(3.0) / sc);
    // ---- Levenberg-Marquardt on the pixel reprojection error (numeric Jacobian, float64)
    int cur = 0;                                           // S.e[cur] holds the residuals at p
    double cost = warp_residual(S, p, f, cx, cy, S.e[0], lane);
    double lambda = 1e-3;
    for (int it = 0; it < 100; ++it) {
        if (lane < 12) {                                   // lane 2j / 2j+1: residuals at p + h_j e_j / p - h_j e_j
            const int j = lane >> 1;
            double pj = p[0];
#pragma unroll
            for (int q = 1; q < 6; ++q) if (q == j) pj = p[q];
            const double h = 1e-6 * fmax(1.0, fabs(pj));
            double pp[6];
#pragma unroll
            for (int q = 0; q < 6; ++q) pp[q] = q == j ? ((lane & 1) ? p[q] - h : p[q] + h) : p[q];
            double Rj[9];
            rodrigues(pp, Rj);
#pragma unroll
            for (int i = 0; i < HP_PTS; ++i) {
                double uv[2];
                project(Rj, pp + 3, S.obj + 3 * i, f, cx, cy, uv);
                S.ep[lane][2 * i] = uv[0] - S.img[2 * i]; S.ep[lane][2 * i + 1] = uv[1] - S.img[2 * i + 1];
            }
            if (!(lane & 1)) S.h[j] = h;
        }
        __syncwarp();
        for (int t = lane; t < 2 * HP_PTS * 6; t += 32) {
            const int i = t / 6, j = t - 6 * i;
            S.J[i][j] = (S.ep[2 * j][i] - S.ep[2 * j + 1][i]) / (2 * S.h[j]);
        }
        __syncwarp();
        for (int t = lane; t < 42; t += 32) {              // J^T J (36 lanes' worth) and J^T e (6)
            double s = 0;
            if (t < 36) {
                const int r = t / 6, c = t - 6 * r;
                for (int i = 0; i < 2 * HP_PTS; ++i) s += S.J[i][r] * S.J[i][c];
                S.JtJ[t] = s;
            } else {
                for (int i = 0; i < 2 * HP_PTS; ++i) s += S.J[i][t - 36] * S.e[cur][i];
                S.Jte[t - 36] = s;
            }
        }
        __syncwarp();
        bool improved = false;
        double step = 0;
        // Raise the damping until a step improves, up to lambda = 1e16 (a gradient step of relative size 1e-16): a fixed
        // number of tries ended small noisy faces at points that were neither stationary nor as good as cv2's.
        while (!improved && lambda <= 1e16) {
            for (int t = lane; t < 42; t += 32) {
                const int r = t / 7, c = t - 7 * r;
                double v;
                if (c == 6) {
                    v = -S.Jte[r];
                } else {
                    v = S.JtJ[r * 6 + c];
                    if (r == c) v += lambda * fmax(v, 1e-12);
                }
                S.Mx[r][c] = v;
            }
            __syncwarp();
            for (int c = 0; c < 6; ++c) {                  // Gaussian elimination with partial pivoting
                int piv = c;
                for (int r = c + 1; r < 6; ++r) if (fabs(S.Mx[r][c]) > fabs(S.Mx[piv][c])) piv = r;
                __syncwarp();
                if (piv != c) {
                    if (lane < 7) { const double t = S.Mx[c][lane]; S.Mx[c][lane] = S.Mx[piv][lane]; S.Mx[piv][lane] = t; }
                    __syncwarp();
                }
                // element (r, q) of the rows below c is t = 7 (r - c - 1) + q: up to 35 of them, so two per lane
                double v[2];
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const int t = lane + 32 * u, r = c + 1 + t / 7, q = t % 7;
                    if (r < 6 && q >= c) {
                        const double mr = S.Mx[r][c] / S.Mx[c][c];
                        v[u] = S.Mx[r][q] - mr * S.Mx[c][q];
                    }
                }
                __syncwarp();
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const int t = lane + 32 * u, r = c + 1 + t / 7, q = t % 7;
                    if (r < 6 && q >= c) S.Mx[r][q] = v[u];
                }
                __syncwarp();
            }
            double dx[6];
#pragma unroll
            for (int r = 5; r >= 0; --r) {
                double s = S.Mx[r][6];
#pragma unroll
                for (int q = r + 1; q < 6; ++q) s -= S.Mx[r][q] * dx[q];
                dx[r] = s / S.Mx[r][r];
            }
            double pn[6];
            for (int q = 0; q < 6; ++q) pn[q] = p[q] + dx[q];
            const double c2 = warp_residual(S, pn, f, cx, cy, S.e[cur ^ 1], lane);
            if (c2 <= cost) {
                step = 0;
                for (int q = 0; q < 6; ++q) { step += dx[q] * dx[q]; p[q] = pn[q]; }
                cur ^= 1;
                cost = c2; lambda = fmax(lambda * 0.1, 1e-15); improved = true;
            } else {
                lambda *= 10;
            }
        }
        if (!improved || step < 1e-24) break;
    }
    // Report the rotation vector with |r| <= pi: shorten the angle by the nearest multiple of 2 pi on the same axis (the
    // iterations may leave it several turns long on small noisy faces).  A round trip through the matrix would do the same
    // but loses up to 2e-5 near theta = pi, where rodrigues_inv rebuilds the axis from the diagonal only (the frontal
    // face [pi, 0, 0] is right there).  r waits in S.h (free once the iterations end) so that it does not stay in
    // registers across rodrigues.
    if (lane == 0) for (int i = 0; i < 3; ++i) S.h[i] = p[i];
    rodrigues(p, R);
    if (lane == 0) {
        const double th = sqrt(S.h[0] * S.h[0] + S.h[1] * S.h[1] + S.h[2] * S.h[2]);
        const double k = th > M_PI ? (th - 2 * M_PI * rint(th / (2 * M_PI))) / th : 1.0;
        for (int i = 0; i < 3; ++i) { a.rvec[(size_t)face * 3 + i] = S.h[i] * k; a.tvec[(size_t)face * 3 + i] = p[3 + i]; }
        euler_rq(R, a.euler + (size_t)face * 3);
    }
    if (lane < 8) project(R, p + 3, S.cube + 3 * lane, f, cx, cy, a.reproj + ((size_t)face * 8 + lane) * 2);
}

void pose_model_98(PoseArgs& a) {
    static const int idx[HP_PTS] = {33, 37, 42, 46, 60, 64, 68, 72, 55, 59};        // headpose.py:64-65
    // the model points and the cube of Skps/core/headpose/pose.py:22-39
    static const float obj[3 * HP_PTS] = {6.825897f, 6.760612f, 4.402142f, 1.330353f, 7.122144f, 6.903745f,
                                          -1.330353f, 7.122144f, 6.903745f, -6.825897f, 6.760612f, 4.402142f,
                                          5.311432f, 5.485328f, 3.987654f, 1.789930f, 5.393625f, 4.413414f,
                                          -1.789930f, 5.393625f, 4.413414f, -5.311432f, 5.485328f, 3.987654f,
                                          2.005628f, 1.409845f, 6.165652f, -2.005628f, 1.409845f, 6.165652f};
    static const float cube[24] = {10, 10, 10, 10, 10, -10, 10, -10, -10, 10, -10, 10,
                                   -10, 10, 10, -10, 10, -10, -10, -10, -10, -10, -10, 10};
    memcpy(a.idx, idx, sizeof(idx));
    memcpy(a.obj, obj, sizeof(obj));
    memcpy(a.cube, cube, sizeof(cube));
}

__global__ void debug_rotation_kernel(const double* r_in, const double* R_in, int n, double* R_out, double* r_out,
                                      double* euler_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    rodrigues(r_in + 3 * (size_t)i, R_out + 9 * (size_t)i);
    rodrigues_inv(R_in + 9 * (size_t)i, r_out + 3 * (size_t)i);
    euler_rq(R_in + 9 * (size_t)i, euler_out + 3 * (size_t)i);
}

int launch_head_pose(const PoseArgs& a, cudaStream_t s) {
    const long long faces = (long long)a.G * a.K;
    if (faces <= 0) return 0;
    head_pose_warp_kernel<<<(unsigned)((faces + HP_WARPS - 1) / HP_WARPS), HP_WARPS * 32, 0, s>>>(a);
    SKPS_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace skps

using namespace skps;

// Batched get_head_pose (pose.py:48-77).  pts [host] (N,10,2) float32 image points in the order of pose.py:60-61
// (landmarks 17,21,22,26,36,39,42,45,31,35 of a 68-point shape); img_w/img_h the frame size (camera matrix of pose.py:50).
// Outputs [host] float64: rvec (N,3), tvec (N,3), euler (N,3) degrees, reproject (N,8,2).
extern "C" SKPS_API int skps_head_pose(const float* pts, int N, int img_w, int img_h, const float* object_pts,
                                       const float* cube_pts, double* rvec, double* tvec, double* euler, double* reproject) {
    SKPS_CHECK(pts && object_pts && cube_pts && rvec && tvec && euler && reproject && N > 0, "head_pose: bad arguments");
    float* d_pts = nullptr;
    double* d_out = nullptr;
    SKPS_CUDA(cudaMalloc(&d_pts, (size_t)N * 2 * HP_PTS * 4));
    if (cudaMalloc(&d_out, (size_t)N * 25 * 8) != cudaSuccess) {
        cudaFree(d_pts);
        SKPS_CHECK(false, "head_pose: cannot allocate the outputs of %d faces", N);
    }
    PoseArgs a = {};
    a.pts32 = d_pts; a.G = 1; a.K = N; a.P = HP_PTS;
    for (int i = 0; i < HP_PTS; ++i) a.idx[i] = i;
    a.H = img_h; a.W = img_w;
    memcpy(a.obj, object_pts, sizeof(a.obj));
    memcpy(a.cube, cube_pts, sizeof(a.cube));
    a.rvec = d_out; a.tvec = d_out + (size_t)N * 3; a.euler = d_out + (size_t)N * 6; a.reproj = d_out + (size_t)N * 9;
    int rc = cudaMemcpy(d_pts, pts, (size_t)N * 2 * HP_PTS * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
             launch_head_pose(a, 0) ||
             cudaMemcpy(rvec, a.rvec, (size_t)N * 24, cudaMemcpyDeviceToHost) != cudaSuccess ||
             cudaMemcpy(tvec, a.tvec, (size_t)N * 24, cudaMemcpyDeviceToHost) != cudaSuccess ||
             cudaMemcpy(euler, a.euler, (size_t)N * 24, cudaMemcpyDeviceToHost) != cudaSuccess ||
             cudaMemcpy(reproject, a.reproj, (size_t)N * 128, cudaMemcpyDeviceToHost) != cudaSuccess;
    const cudaError_t err = cudaGetLastError();
    cudaFree(d_pts); cudaFree(d_out);
    SKPS_CHECK(!rc, "head_pose: %s", err == cudaSuccess ? get_error() : cudaGetErrorString(err));
    return 0;
}

// The solver's rotation helpers on their own, in device code: R_out[i] = rodrigues(r_in[i]); r_out[i] = rodrigues_inv(R_in[i]);
// euler_out[i] = euler_rq(R_in[i]).  r_in (n,3), R_in (n,3,3) row-major, all [host] float64.
extern "C" SKPS_API int skps_debug_rotation(const double* r_in, const double* R_in, int n, double* R_out, double* r_out,
                                            double* euler_out) {
    SKPS_CHECK(r_in && R_in && R_out && r_out && euler_out && n > 0, "debug_rotation: bad arguments");
    double* d = nullptr;
    SKPS_CUDA(cudaMalloc(&d, (size_t)n * 30 * 8));
    double *dr = d, *dR = d + (size_t)n * 3, *dRo = d + (size_t)n * 12, *dro = d + (size_t)n * 21, *de = d + (size_t)n * 24;
    int rc = cudaMemcpy(dr, r_in, (size_t)n * 24, cudaMemcpyHostToDevice) != cudaSuccess ||
             cudaMemcpy(dR, R_in, (size_t)n * 72, cudaMemcpyHostToDevice) != cudaSuccess;
    cudaError_t err = cudaSuccess;
    if (!rc) {
        debug_rotation_kernel<<<(n + 127) / 128, 128>>>(dr, dR, n, dRo, dro, de);
        err = cudaGetLastError();
        if (err == cudaSuccess) err = cudaMemcpy(R_out, dRo, (size_t)n * 72, cudaMemcpyDeviceToHost);
        if (err == cudaSuccess) err = cudaMemcpy(r_out, dro, (size_t)n * 24, cudaMemcpyDeviceToHost);
        if (err == cudaSuccess) err = cudaMemcpy(euler_out, de, (size_t)n * 24, cudaMemcpyDeviceToHost);
    }
    cudaFree(d);
    SKPS_CHECK(!rc && err == cudaSuccess, "debug_rotation: %s", rc ? "cannot copy the inputs" : cudaGetErrorString(err));
    return 0;
}
