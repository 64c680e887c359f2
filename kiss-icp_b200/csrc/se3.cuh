// SE(3)/SO(3) arithmetic for the device path (and the host side of the C-ABI).
//
// The reference does this arithmetic through Sophus 1.24.6 and Eigen 3.4.0 (not vendored in
// the reference tree). The formulas below follow the published algorithms of those versions
// at the call sites of the hot path:
//   SE3::exp / log            cpp/kiss_icp/core/Registration.cpp:157, Preprocessing.cpp:68,78
//   SE3 * point / SE3 * SE3   Registration.cpp:57,161,166; VoxelHashMap.cpp:92; KissICP.cpp:47,57,62
//   Matrix6d::ldlt().solve    Registration.cpp:156
//   AngleAxisd(R).angle()     Threshold.cpp:40
// Everything is FP64 like the reference. The file is compiled with -fmad=false so that
// products and sums round exactly like the x86-64 reference build (no FMA contraction).
#pragma once

#include <cfloat>
#include <cmath>

#include "types.cuh"

#define KB_HD __host__ __device__ __forceinline__

namespace kb {

using kb_types::Q4;
using kb_types::SE3;
using kb_types::V3;

KB_HD V3 operator+(const V3 &a, const V3 &b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
KB_HD V3 operator-(const V3 &a, const V3 &b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
KB_HD V3 operator*(double s, const V3 &a) { return {s * a.x, s * a.y, s * a.z}; }
KB_HD V3 cross(const V3 &a, const V3 &b) {
    return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
KB_HD double sqnorm(const V3 &a) { return (a.x * a.x + a.y * a.y) + a.z * a.z; }
KB_HD double norm(const V3 &a) { return sqrt(sqnorm(a)); }

// _correct_kitti_scan for one point (kiss_icp_pybind.cpp:127-138): rotate by the fixed angle about
// normalized(pt x e_z), evaluated like Eigen's AngleAxisd::toRotationMatrix() * pt; sn, cs = sin / cos of the angle
KB_HD V3 correct_kitti_point(const V3 &pt, double sn, double cs) {
    V3 ax = cross(pt, V3{0.0, 0.0, 1.0});
    const double z = sqnorm(ax);
    if (z > 0.0) {
        const double n = sqrt(z);
        ax = V3{ax.x / n, ax.y / n, ax.z / n};
    }
    const V3 sa{sn * ax.x, sn * ax.y, sn * ax.z};
    const double c1 = 1.0 - cs;
    const V3 ca{c1 * ax.x, c1 * ax.y, c1 * ax.z};
    double t = ca.x * ax.y;
    const double r01 = t - sa.z, r10 = t + sa.z;
    t = ca.x * ax.z;
    const double r02 = t + sa.y, r20 = t - sa.y;
    t = ca.y * ax.z;
    const double r12 = t - sa.x, r21 = t + sa.x;
    const double r00 = ca.x * ax.x + cs, r11 = ca.y * ax.y + cs, r22 = ca.z * ax.z + cs;
    return V3{(r00 * pt.x + r01 * pt.y) + r02 * pt.z, (r10 * pt.x + r11 * pt.y) + r12 * pt.z,
              (r20 * pt.x + r21 * pt.y) + r22 * pt.z};
}

KB_HD SE3 se3_identity() { return SE3{{0, 0, 0, 1}, {0, 0, 0}}; }

constexpr double kEps = 1e-10;  // Sophus::Constants<double>::epsilon()
constexpr double kSchurNoise = 0x1p-42;  // 1024 DBL_EPSILON: icp_solve_schur's floor under cancellation

KB_HD Q4 q_normalized(const Q4 &q) {
    const double len = sqrt(((q.x * q.x + q.y * q.y) + q.z * q.z) + q.w * q.w);
    return {q.x / len, q.y / len, q.z / len, q.w / len};
}

KB_HD Q4 q_mul(const Q4 &a, const Q4 &b) {
    Q4 r;
    r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
    r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
    r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
    r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
    return q_normalized(r);
}

// v + w*(2 q x v) + q x (2 q x v)
KB_HD V3 q_rotate(const Q4 &q, const V3 &v) {
    const V3 qv{q.x, q.y, q.z};
    V3 uv = cross(qv, v);
    uv = uv + uv;
    return (v + q.w * uv) + cross(qv, uv);
}

KB_HD V3 se3_act(const SE3 &T, const V3 &p) { return q_rotate(T.q, p) + T.t; }

KB_HD SE3 se3_mul(const SE3 &a, const SE3 &b) {
    SE3 r;
    r.q = q_mul(a.q, b.q);
    r.t = a.t + q_rotate(a.q, b.t);
    return r;
}

KB_HD SE3 se3_inverse(const SE3 &a) {
    SE3 r;
    r.q = q_normalized(Q4{-a.q.x, -a.q.y, -a.q.z, a.q.w});
    r.t = q_rotate(r.q, V3{a.t.x * -1.0, a.t.y * -1.0, a.t.z * -1.0});
    return r;
}

struct M3 {
    double m[3][3];
};

KB_HD M3 q_to_matrix(const Q4 &q) {
    const double tx = 2.0 * q.x, ty = 2.0 * q.y, tz = 2.0 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    M3 r;
    r.m[0][0] = 1.0 - (tyy + tzz);
    r.m[0][1] = txy - twz;
    r.m[0][2] = txz + twy;
    r.m[1][0] = txy + twz;
    r.m[1][1] = 1.0 - (txx + tzz);
    r.m[1][2] = tyz - twx;
    r.m[2][0] = txz - twy;
    r.m[2][1] = tyz + twx;
    r.m[2][2] = 1.0 - (txx + tyy);
    return r;
}

// quaternion from rotation matrix (Shoemake), as Eigen does for Quaterniond(Matrix3d)
KB_HD Q4 q_from_matrix(const M3 &mat) {
    double c[4];
    double t = mat.m[0][0] + mat.m[1][1] + mat.m[2][2];
    if (t > 0.0) {
        t = sqrt(t + 1.0);
        c[3] = 0.5 * t;
        t = 0.5 / t;
        c[0] = (mat.m[2][1] - mat.m[1][2]) * t;
        c[1] = (mat.m[0][2] - mat.m[2][0]) * t;
        c[2] = (mat.m[1][0] - mat.m[0][1]) * t;
    } else {
        int i = 0;
        if (mat.m[1][1] > mat.m[0][0]) i = 1;
        if (mat.m[2][2] > mat.m[i][i]) i = 2;
        const int j = (i + 1) % 3;
        const int k = (j + 1) % 3;
        t = sqrt(mat.m[i][i] - mat.m[j][j] - mat.m[k][k] + 1.0);
        c[i] = 0.5 * t;
        t = 0.5 / t;
        c[3] = (mat.m[k][j] - mat.m[j][k]) * t;
        c[j] = (mat.m[j][i] + mat.m[i][j]) * t;
        c[k] = (mat.m[k][i] + mat.m[i][k]) * t;
    }
    return {c[0], c[1], c[2], c[3]};
}

KB_HD Q4 so3_exp(const V3 &omega, double *theta_out) {
    const double theta_sq = sqnorm(omega);
    double imag_factor, real_factor, theta;
    if (theta_sq < kEps * kEps) {
        theta = 0.0;
        const double theta_po4 = theta_sq * theta_sq;
        imag_factor = 0.5 - (1.0 / 48.0) * theta_sq + (1.0 / 3840.0) * theta_po4;
        real_factor = 1.0 - (1.0 / 8.0) * theta_sq + (1.0 / 384.0) * theta_po4;
    } else {
        theta = sqrt(theta_sq);
        const double half_theta = 0.5 * theta;
        imag_factor = sin(half_theta) / theta;
        real_factor = cos(half_theta);
    }
    *theta_out = theta;
    return {imag_factor * omega.x, imag_factor * omega.y, imag_factor * omega.z, real_factor};
}

KB_HD V3 so3_log(const Q4 &q, double *theta_out) {
    const double squared_n = (q.x * q.x + q.y * q.y) + q.z * q.z;
    const double w = q.w;
    double two_atan_nbyw_by_n, theta;
    if (squared_n < kEps * kEps) {
        const double squared_w = w * w;
        two_atan_nbyw_by_n = 2.0 / w - (2.0 / 3.0) * (squared_n) / (w * squared_w);
        theta = 2.0 * squared_n / w;
    } else {
        const double n = sqrt(squared_n);
        const double atan_nbyw = (w < 0.0) ? atan2(-n, -w) : atan2(n, w);
        two_atan_nbyw_by_n = 2.0 * atan_nbyw / n;
        theta = two_atan_nbyw_by_n * n;
    }
    *theta_out = theta;
    return {two_atan_nbyw_by_n * q.x, two_atan_nbyw_by_n * q.y, two_atan_nbyw_by_n * q.z};
}

// y = (I + a*hat(w) + b*hat(w)^2) v, with the same matrix-entry arithmetic as the dense form
KB_HD V3 apply_I_aW_bW2(const V3 &w, double a, double b, bool use_b, const V3 &v) {
    // Omega = hat(w); Omega_sq = Omega*Omega (each entry (p0+p1)+p2 with exact zeros)
    const double O[3][3] = {{0.0, -w.z, w.y}, {w.z, 0.0, -w.x}, {-w.y, w.x, 0.0}};
    double O2[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) O2[i][j] = (O[i][0] * O[0][j] + O[i][1] * O[1][j]) + O[i][2] * O[2][j];
    double V[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            const double id = (i == j) ? 1.0 : 0.0;
            V[i][j] = use_b ? ((id + a * O[i][j]) + b * O2[i][j]) : (id + a * O[i][j]);
        }
    return {(V[0][0] * v.x + V[0][1] * v.y) + V[0][2] * v.z, (V[1][0] * v.x + V[1][1] * v.y) + V[1][2] * v.z,
            (V[2][0] * v.x + V[2][1] * v.y) + V[2][2] * v.z};
}

// Sophus SE3::exp, tangent = (upsilon, omega)
KB_HD SE3 se3_exp(const double a[6]) {
    const V3 upsilon{a[0], a[1], a[2]};
    const V3 omega{a[3], a[4], a[5]};
    double theta;
    SE3 r;
    r.q = so3_exp(omega, &theta);
    const double theta_sq = theta * theta;
    if (theta_sq < kEps * kEps) {
        r.t = apply_I_aW_bW2(omega, 0.5, 0.0, false, upsilon);
    } else {
        const double ca = (1.0 - cos(theta)) / theta_sq;
        const double cb = (theta - sin(theta)) / (theta_sq * theta);
        r.t = apply_I_aW_bW2(omega, ca, cb, true, upsilon);
    }
    return r;
}

// Sophus SE3::log
KB_HD void se3_log(const SE3 &T, double out[6]) {
    double theta;
    const V3 omega = so3_log(T.q, &theta);
    V3 u;
    if (fabs(theta) < kEps) {
        u = apply_I_aW_bW2(omega, -0.5, 1. / 12., true, T.t);
    } else {
        const double half_theta = 0.5 * theta;
        const double c = (1.0 - theta * cos(half_theta) / (2.0 * sin(half_theta))) / (theta * theta);
        u = apply_I_aW_bW2(omega, -0.5, c, true, T.t);
    }
    out[0] = u.x;
    out[1] = u.y;
    out[2] = u.z;
    out[3] = omega.x;
    out[4] = omega.y;
    out[5] = omega.z;
}

// A sampled trajectory (kb_motion, DESIGN.md section 4.17) is T(t) = T_k Exp(tau xi_k) on interval k, tau = t - t_k,
// xi_k = Log(T_k^-1 T_k+1) / (t_k+1 - t_k). motion_interval: the k in [0, m - 2] of t among the m sample times
// times[0], times[stride], ...; before the first and after the last sample the first and the last interval (they are
// extrapolated), and 0 for a NaN t.
KB_HD int motion_interval(const double *times, int stride, int m, double t) {
    int lo = 0, hi = m - 1;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (times[mid * stride] <= t)
            lo = mid;
        else
            hi = mid;
    }
    return lo;
}
KB_HD SE3 motion_at(const SE3 &Tk, const double xi[6], double tau) {
    double a[6];
    for (int i = 0; i < 6; ++i) a[i] = tau * xi[i];
    return se3_mul(Tk, se3_exp(a));
}

// Eigen::AngleAxisd(Matrix3d).angle()
KB_HD double angle_axis_angle(const M3 &R) {
    const Q4 q = q_from_matrix(R);
    double n = sqrt((q.x * q.x + q.y * q.y) + q.z * q.z);
    if (n < DBL_EPSILON) {
        const double m = fmax(fabs(q.x), fmax(fabs(q.y), fabs(q.z)));
        if (m > 0.0) {
            const double a = q.x / m, b = q.y / m, c = q.z / m;
            n = m * sqrt((a * a + b * b) + c * c);
        } else {
            n = 0.0;
        }
    }
    if (n != 0.0) return 2.0 * atan2(n, fabs(q.w));
    return 0.0;
}

// row-major 4x4 -> SE3; false where Sophus would fail its orthogonality / last-row checks
KB_HD bool se3_from_matrix(const double M[16], SE3 *out) {
    M3 R;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) R.m[i][j] = M[4 * i + j];
    double fro = 0.0;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double s = 0.0;
            for (int k = 0; k < 3; ++k) s += R.m[i][k] * R.m[j][k];
            s -= (i == j) ? 1.0 : 0.0;
            fro += s * s;
        }
    const double det = R.m[0][0] * (R.m[1][1] * R.m[2][2] - R.m[1][2] * R.m[2][1]) -
                       R.m[0][1] * (R.m[1][0] * R.m[2][2] - R.m[1][2] * R.m[2][0]) +
                       R.m[0][2] * (R.m[1][0] * R.m[2][1] - R.m[1][1] * R.m[2][0]);
    if (!(sqrt(fro) < kEps) || !(det > 0.0)) return false;
    if (!(fabs(M[12]) < kEps && fabs(M[13]) < kEps && fabs(M[14]) < kEps && fabs(M[15] - 1.0) < kEps)) return false;
    out->q = q_from_matrix(R);
    out->t = {M[3], M[7], M[11]};
    return true;
}

KB_HD void se3_to_matrix(const SE3 &T, double M[16]) {
    const M3 R = q_to_matrix(T.q);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) M[4 * i + j] = R.m[i][j];
    M[3] = T.t.x;
    M[7] = T.t.y;
    M[11] = T.t.z;
    M[12] = M[13] = M[14] = 0.0;
    M[15] = 1.0;
}

// Pieces of ldlt6_solve_fast (below): LDL^T with diagonal pivoting of a symmetric 6x6 following Eigen 3.4 LDLT (Lower,
// unblocked), first-max pivot. Every index is resolved at compile time (a pivot swap is expanded into one guarded block
// per possible pivot row), so the 6x6 lives in registers instead of local memory.
template <int K, int BIG>
KB_HD void ldlt6_swap(double (&mat)[6][6]) {
    constexpr int N = 6;
    constexpr int S = N - BIG - 1;
#pragma unroll
    for (int j = 0; j < K; ++j) {
        const double t = mat[K][j];
        mat[K][j] = mat[BIG][j];
        mat[BIG][j] = t;
    }
#pragma unroll
    for (int i = 0; i < S; ++i) {
        const double t = mat[N - S + i][K];
        mat[N - S + i][K] = mat[N - S + i][BIG];
        mat[N - S + i][BIG] = t;
    }
    {
        const double t = mat[K][K];
        mat[K][K] = mat[BIG][BIG];
        mat[BIG][BIG] = t;
    }
#pragma unroll
    for (int i = K + 1; i < BIG; ++i) {
        const double t = mat[i][K];
        mat[i][K] = mat[BIG][i];
        mat[BIG][i] = t;
    }
}

template <int K>
KB_HD void ldlt6_apply_tr(double (&d)[6], int big) {
#pragma unroll
    for (int b = K + 1; b < 6; ++b)
        if (big == b) {
            const double t = d[K];
            d[K] = d[b];
            d[b] = t;
        }
}

// ---- latency-optimised variants for the ICP inner loop -------------------------------------
// The ICP solve is a single-thread dependent chain executed once per iteration; a DDIV, DSQRT
// or sin/cos costs an order of magnitude more latency than a DADD/DMUL (tools/latency_probe.cu
// measures them). The LDL^T multiplies by ONE reciprocal per pivot where Eigen's divides, and
// se3_exp_fast takes one sincos(theta/2) with double-angle identities instead of se3_exp's four
// separate sin/cos calls. They differ from Eigen's LDLT and from se3_exp / se3_mul by a few ulps
// (tests bound the difference against the oracle) — far inside the 1e-4 m / 1e-4 rad parity budget.
// ~1-ulp reciprocal: MUFU seed (rcp.approx.ftz.f64, ~20 bits) + two Newton steps in FMA —
// a fraction of the latency of an IEEE DDIV (host: plain division).
KB_HD double fast_rcp(double x) {
#ifdef __CUDA_ARCH__
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
    r = fma(r, fma(-x, r, 1.0), r);
    r = fma(r, fma(-x, r, 1.0), r);
    return r;
#else
    return 1.0 / x;
#endif
}

template <int K>
KB_HD bool ldlt6_step_fast(double (&mat)[6][6], int (&tr)[6], double (&inv)[6]) {
    constexpr int N = 6;
    int big = K;
    double best = fabs(mat[K][K]);
#pragma unroll
    for (int i = K + 1; i < N; ++i) {
        const double v = fabs(mat[i][i]);
        if (v > best) {
            best = v;
            big = i;
        }
    }
    tr[K] = big;
    if (K + 1 < N && big == K + 1) ldlt6_swap<K, (K + 1 < N ? K + 1 : K)>(mat);
    if (K + 2 < N && big == K + 2) ldlt6_swap<K, (K + 2 < N ? K + 2 : K)>(mat);
    if (K + 3 < N && big == K + 3) ldlt6_swap<K, (K + 3 < N ? K + 3 : K)>(mat);
    if (K + 4 < N && big == K + 4) ldlt6_swap<K, (K + 4 < N ? K + 4 : K)>(mat);
    if (K + 5 < N && big == K + 5) ldlt6_swap<K, (K + 5 < N ? K + 5 : K)>(mat);
    constexpr int RS = N - K - 1;
    if (K > 0) {
        double temp[6];
#pragma unroll
        for (int j = 0; j < K; ++j) temp[j] = mat[j][j] * mat[K][j];
        double acc = 0.0;
#pragma unroll
        for (int j = 0; j < K; ++j) acc += mat[K][j] * temp[j];
        mat[K][K] -= acc;
#pragma unroll
        for (int i = 0; i < RS; ++i) {
            double a2 = 0.0;
#pragma unroll
            for (int j = 0; j < K; ++j) a2 += mat[K + 1 + i][j] * temp[j];
            mat[K + 1 + i][K] -= a2;
        }
    }
    const double akk = mat[K][K];
    const bool valid = fabs(akk) > 0.0;
    if (K == 0 && !valid) return false;
    const double r = (fabs(akk) > 1e-290 && fabs(akk) < 1e290) ? fast_rcp(akk) : (valid ? 1.0 / akk : 0.0);
    inv[K] = (fabs(akk) > DBL_MIN) ? r : 0.0;  // D^+ of the solve (pivots <= DBL_MIN give 0)
    if (RS > 0 && valid) {
#pragma unroll
        for (int i = 0; i < RS; ++i) mat[K + 1 + i][K] *= r;
    }
    return true;
}

KB_HD void ldlt6_solve_fast(const double A_in[36], const double b[6], double x[6]) {
    constexpr int N = 6;
    double mat[6][6];
#pragma unroll
    for (int i = 0; i < N; ++i)
#pragma unroll
        for (int j = 0; j < N; ++j) mat[i][j] = A_in[N * i + j];
    int tr[6] = {0, 1, 2, 3, 4, 5};
    double inv[6] = {0, 0, 0, 0, 0, 0};
    if (ldlt6_step_fast<0>(mat, tr, inv)) {
        ldlt6_step_fast<1>(mat, tr, inv);
        ldlt6_step_fast<2>(mat, tr, inv);
        ldlt6_step_fast<3>(mat, tr, inv);
        ldlt6_step_fast<4>(mat, tr, inv);
        ldlt6_step_fast<5>(mat, tr, inv);
    } else {
        tr[0] = 0;
    }
    double d[6];
#pragma unroll
    for (int i = 0; i < N; ++i) d[i] = b[i];
    ldlt6_apply_tr<0>(d, tr[0]);
    ldlt6_apply_tr<1>(d, tr[1]);
    ldlt6_apply_tr<2>(d, tr[2]);
    ldlt6_apply_tr<3>(d, tr[3]);
    ldlt6_apply_tr<4>(d, tr[4]);
#pragma unroll
    for (int i = 0; i < N; ++i) {
        double acc = d[i];
#pragma unroll
        for (int j = 0; j < i; ++j) acc -= mat[i][j] * d[j];
        d[i] = acc;
    }
#pragma unroll
    for (int i = 0; i < N; ++i) d[i] *= inv[i];
#pragma unroll
    for (int i = N - 1; i >= 0; --i) {
        double acc = d[i];
#pragma unroll
        for (int j = i + 1; j < N; ++j) acc -= mat[j][i] * d[j];
        d[i] = acc;
    }
    ldlt6_apply_tr<4>(d, tr[4]);
    ldlt6_apply_tr<3>(d, tr[3]);
    ldlt6_apply_tr<2>(d, tr[2]);
    ldlt6_apply_tr<1>(d, tr[1]);
    ldlt6_apply_tr<0>(d, tr[0]);
#pragma unroll
    for (int i = 0; i < N; ++i) x[i] = d[i];
}

// SE3::exp for a small rotation (kEps^2 <= |omega|^2 < 0.01).
// ICP steps are tiny rotations: sin(t/2)/t, cos(t/2), (1 - cos t)/t^2 and (t - sin t)/t^3 are even power series
// in t — evaluated in t^2 (Horner, FMA) there is no square root, no division and no sincos on the solver's
// dependent chain. Truncation < 1e-19 relative for t < 0.1 rad.
KB_HD SE3 se3_exp_small(const double a[6], double theta_sq) {
    const V3 upsilon{a[0], a[1], a[2]};
    const V3 omega{a[3], a[4], a[5]};
    SE3 r;
    const double h2 = 0.25 * theta_sq;  // (t/2)^2
    const double sinc = fma(h2, fma(h2, fma(h2, fma(h2, fma(h2, -1.0 / 39916800.0, 1.0 / 362880.0), -1.0 / 5040.0), 1.0 / 120.0), -1.0 / 6.0), 1.0);
    const double ch = fma(h2, fma(h2, fma(h2, fma(h2, fma(h2, fma(h2, 1.0 / 479001600.0, -1.0 / 3628800.0), 1.0 / 40320.0), -1.0 / 720.0), 1.0 / 24.0), -0.5), 1.0);
    const double imag = 0.5 * sinc;  // sin(t/2) / t
    r.q = Q4{imag * omega.x, imag * omega.y, imag * omega.z, ch};
    const double t2 = theta_sq;
    const double ca = fma(t2, fma(t2, fma(t2, fma(t2, fma(t2, -1.0 / 479001600.0, 1.0 / 3628800.0), -1.0 / 40320.0), 1.0 / 720.0), -1.0 / 24.0), 0.5);
    const double cb = fma(t2, fma(t2, fma(t2, fma(t2, fma(t2, -1.0 / 6227020800.0, 1.0 / 39916800.0), -1.0 / 362880.0), 1.0 / 5040.0), -1.0 / 120.0), 1.0 / 6.0);
    r.t = apply_I_aW_bW2(omega, ca, cb, true, upsilon);
    return r;
}

KB_HD SE3 se3_exp_fast(const double a[6]) {
    const V3 upsilon{a[0], a[1], a[2]};
    const V3 omega{a[3], a[4], a[5]};
    const double theta_sq = sqnorm(omega);
    SE3 r;
    if (theta_sq < kEps * kEps) return se3_exp(a);
    if (theta_sq < 0.01) return se3_exp_small(a, theta_sq);
    const double theta = sqrt(theta_sq);
    const double inv_theta = fast_rcp(theta);
    double sh, ch;
    sincos(0.5 * theta, &sh, &ch);
    const double imag = sh * inv_theta;
    r.q = Q4{imag * omega.x, imag * omega.y, imag * omega.z, ch};
    // (1 - cos t)/t^2 = 2 sin^2(t/2)/t^2 ;  (t - sin t)/t^3 with sin t = 2 sin(t/2) cos(t/2)
    const double ca = 2.0 * imag * imag;
    const double cb = (theta - 2.0 * sh * ch) * (inv_theta * inv_theta * inv_theta);
    r.t = apply_I_aW_bW2(omega, ca, cb, true, upsilon);
    return r;
}

KB_HD SE3 se3_mul_fast(const SE3 &a, const SE3 &b) {
    Q4 q;
    q.w = a.q.w * b.q.w - a.q.x * b.q.x - a.q.y * b.q.y - a.q.z * b.q.z;
    q.x = a.q.w * b.q.x + a.q.x * b.q.w + a.q.y * b.q.z - a.q.z * b.q.y;
    q.y = a.q.w * b.q.y + a.q.y * b.q.w + a.q.z * b.q.x - a.q.x * b.q.z;
    q.z = a.q.w * b.q.z + a.q.z * b.q.w + a.q.x * b.q.y - a.q.y * b.q.x;
    const double inv_len = 1.0 / sqrt(((q.x * q.x + q.y * q.y) + q.z * q.z) + q.w * q.w);
    SE3 r;
    r.q = Q4{q.x * inv_len, q.y * inv_len, q.z * inv_len, q.w * inv_len};
    r.t = a.t + q_rotate(a.q, b.t);
    return r;
}

// ---- structured solve of the ICP normal equations ------------------------------------------
// With J = [I | -hat(s)] the 6x6 system is  [ a I   B^T ] [x1]   [r1]      a = sum w,  B = hat(m), m = sum w s,
//                                           [ B     C   ] [x2] = [r2]      C = sum w hat(s)^T hat(s)
// so x2 solves the 3x3 Schur complement  S x2 = r2 - (m x r1)/a,  S = C + (m m^T - |m|^2 I)/a,  and
// x1 = (r1 + m x x2)/a. ~90 flops and two reciprocals instead of a pivoted 6x6 LDL^T (thousands of cycles of
// dependent FP64 work): the same linear system, a different rounding path (like the reference's own
// nondeterministic summation order). Returns false (caller falls back to the LDL^T) when the system is
// degenerate: no correspondences, or a Schur complement that is not safely invertible.
KB_HD bool icp_solve_schur(const double acc[16], double dx[6]) {
    const double a = acc[0];
    if (!(a > 1e-300)) return false;
    const double inv_a = fast_rcp(a);
    const V3 m{acc[1], acc[2], acc[3]};
    // rhs = -JTr
    const V3 r1{-acc[10], -acc[11], -acc[12]};
    const V3 r2{-acc[13], -acc[14], -acc[15]};
    // C (symmetric): (3,3) (4,3) (4,4) (5,3) (5,4) (5,5) = acc[4..9]
    const double mm = sqnorm(m);
    const double s00 = acc[4] + (m.x * m.x - mm) * inv_a;
    const double s10 = acc[5] + (m.y * m.x) * inv_a;
    const double s11 = acc[6] + (m.y * m.y - mm) * inv_a;
    const double s20 = acc[7] + (m.z * m.x) * inv_a;
    const double s21 = acc[8] + (m.z * m.y) * inv_a;
    const double s22 = acc[9] + (m.z * m.z - mm) * inv_a;
    const V3 mxr1 = cross(m, r1);
    const V3 b{r2.x - mxr1.x * inv_a, r2.y - mxr1.y * inv_a, r2.z - mxr1.z * inv_a};
    // adjugate of the symmetric 3x3
    const double c00 = s11 * s22 - s21 * s21;
    const double c01 = s20 * s21 - s10 * s22;
    const double c02 = s10 * s21 - s20 * s11;
    const double c11 = s00 * s22 - s20 * s20;
    const double c12 = s10 * s20 - s00 * s21;
    const double c22 = s00 * s11 - s10 * s10;
    const double det = s00 * c00 + s10 * c01 + s20 * c02;
    const double scale = (fabs(s00) + fabs(s11) + fabs(s22)) * (1.0 / 3.0);
    // S is C minus terms as large as C. Where they cancel in exact arithmetic (one correspondence, coincident points,
    // points on one line) what is left is their rounding, ~eps tr(C), and the relative test above compares that noise
    // with itself. So S, and det S against scale^2, must also stand above kSchurNoise tr(C)/3: 1024 eps, 30x the
    // rounding measured on 2000 sequentially summed correspondences (DESIGN.md, "Degenerate systems").
    const double noise = kSchurNoise * (((acc[4] + acc[6]) + acc[9]) * (1.0 / 3.0));
    if (!(fabs(det) > 1e-9 * scale * scale * scale) || !(scale > 0.0) || !(scale > noise) ||
        !(fabs(det) > noise * scale * scale))
        return false;
    const double inv_det = fast_rcp(det);
    const V3 x2{(c00 * b.x + c01 * b.y + c02 * b.z) * inv_det, (c01 * b.x + c11 * b.y + c12 * b.z) * inv_det,
                (c02 * b.x + c12 * b.y + c22 * b.z) * inv_det};
    const V3 mxx2 = cross(m, x2);
    dx[0] = (r1.x + mxx2.x) * inv_a;
    dx[1] = (r1.y + mxx2.y) * inv_a;
    dx[2] = (r1.z + mxx2.z) * inv_a;
    dx[3] = x2.x;
    dx[4] = x2.y;
    dx[5] = x2.z;
    return true;
}

// ---- Jacobians of the pose graph (kb_pose_graph_optimize) -------------------------------------------------------------
// Tangent order (translation, rotation), as se3_exp / se3_log; 6x6 matrices row-major.
// Ad(T) = [R, hat(t) R; 0, R]: T Exp(x) T^-1 = Exp(Ad(T) x).
KB_HD void se3_adjoint(const SE3 &T, double A[36]) {
    const M3 R = q_to_matrix(T.q);
    const double th[3][3] = {{0.0, -T.t.z, T.t.y}, {T.t.z, 0.0, -T.t.x}, {-T.t.y, T.t.x, 0.0}};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            A[6 * i + j] = R.m[i][j];
            A[6 * i + j + 3] = (th[i][0] * R.m[0][j] + th[i][1] * R.m[1][j]) + th[i][2] * R.m[2][j];
            A[6 * (i + 3) + j] = 0.0;
            A[6 * (i + 3) + j + 3] = R.m[i][j];
        }
}

KB_HD void m3_mul(const double a[3][3], const double b[3][3], double c[3][3]) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) c[i][j] = (a[i][0] * b[0][j] + a[i][1] * b[1][j]) + a[i][2] * b[2][j];
}

// J_r^-1(x): Log(Exp(x) Exp(d)) = x + J_r^-1(x) d + O(|d|^2). J_r^-1(x) = J_l^-1(-x), with (rho, phi) = -x,
//   J_l^-1 = [S, -S Q S; 0, S],  S = I - hat(phi)/2 + c hat(phi)^2,  c = 1/t^2 - (1 + cos t) / (2 t sin t),  t = |phi|,
//   Q = hat(rho)/2 + c1 (P Rh + Rh P + P Rh P) + c2 (P P Rh + Rh P P - 3 P Rh P) + c3 (P Rh P P + P P Rh P),
//   P = hat(phi), Rh = hat(rho), c1 = (t - sin t)/t^3, c2 = (t^2 + 2 cos t - 2)/(2 t^4), c3 = (2 t - 3 sin t + t cos t)/(2 t^5)
//   (Barfoot, State Estimation for Robotics, 7.1.5). Below t = 0.5 the coefficients are their Taylor series to t^12
//   (truncation below 1e-17 absolute): the closed forms of c1, c2 and c3 cancel there, c2's by eps / t^4 relative. c is
//   evaluated as 1/t^2 - cot(t/2) / (2t): the equal (1 + cos t) / (2 t sin t) loses 1 + cos t near t = pi. Measured
//   against a 60-digit Log(Exp(x) Exp(d)) for |rho| up to 100 and t from 0 to pi - 1e-7: within 1e-15 of max |J|
//   (tests/test_pose_graph_shapes.py).
KB_HD void se3_right_jacobian_inverse(const double x[6], double J[36]) {
    const double rho[3] = {-x[0], -x[1], -x[2]}, phi[3] = {-x[3], -x[4], -x[5]};
    const double t2 = (phi[0] * phi[0] + phi[1] * phi[1]) + phi[2] * phi[2];
    double c, c1, c2, c3;
    if (t2 < 0.25) {
        // (Horner in t^2; c's coefficients are B_{2k+2} / (2k+2)! in magnitude, Bernoulli numbers)
        c = 1.0 / 12.0 + t2 * (1.0 / 720.0 + t2 * (1.0 / 30240.0 + t2 * (1.0 / 1209600.0 + t2 * (1.0 / 47900160.0 +
            t2 * (691.0 / 1307674368000.0 + t2 * (1.0 / 74724249600.0))))));
        c1 = 1.0 / 6.0 - t2 * (1.0 / 120.0 - t2 * (1.0 / 5040.0 - t2 * (1.0 / 362880.0 - t2 * (1.0 / 39916800.0 -
             t2 * (1.0 / 6227020800.0 - t2 * (1.0 / 1307674368000.0))))));
        c2 = 1.0 / 24.0 - t2 * (1.0 / 720.0 - t2 * (1.0 / 40320.0 - t2 * (1.0 / 3628800.0 - t2 * (1.0 / 479001600.0 -
             t2 * (1.0 / 87178291200.0 - t2 * (1.0 / 20922789888000.0))))));
        c3 = 1.0 / 120.0 - t2 * (1.0 / 2520.0 - t2 * (1.0 / 120960.0 - t2 * (1.0 / 9979200.0 - t2 * (1.0 / 1245404160.0 -
             t2 * (1.0 / 217945728000.0 - t2 * (1.0 / 50812489728000.0))))));
    } else {
        const double t = sqrt(t2), st = sin(t), ct = cos(t), h = 0.5 * t;
        c = 1.0 / t2 - cos(h) / (2.0 * t * sin(h));
        c1 = (t - st) / (t2 * t);
        c2 = ((t2 + 2.0 * ct) - 2.0) / (2.0 * t2 * t2);
        c3 = ((2.0 * t - 3.0 * st) + t * ct) / (2.0 * t2 * t2 * t);
    }
    const double P[3][3] = {{0.0, -phi[2], phi[1]}, {phi[2], 0.0, -phi[0]}, {-phi[1], phi[0], 0.0}};
    const double Rh[3][3] = {{0.0, -rho[2], rho[1]}, {rho[2], 0.0, -rho[0]}, {-rho[1], rho[0], 0.0}};
    double PP[3][3], PR[3][3], RP[3][3], PRP[3][3], PPR[3][3], RPP[3][3], PRPP[3][3], PPRP[3][3];
    m3_mul(P, P, PP);
    m3_mul(P, Rh, PR);
    m3_mul(Rh, P, RP);
    m3_mul(PR, P, PRP);
    m3_mul(PP, Rh, PPR);
    m3_mul(RP, P, RPP);
    m3_mul(PRP, P, PRPP);
    m3_mul(PP, RP, PPRP);
    double S[3][3], Q[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            S[i][j] = ((i == j ? 1.0 : 0.0) - 0.5 * P[i][j]) + c * PP[i][j];
            Q[i][j] = ((0.5 * Rh[i][j] + c1 * ((PR[i][j] + RP[i][j]) + PRP[i][j])) +
                       c2 * ((PPR[i][j] + RPP[i][j]) - 3.0 * PRP[i][j])) +
                      c3 * (PRPP[i][j] + PPRP[i][j]);
        }
    double SQ[3][3], SQS[3][3];
    m3_mul(S, Q, SQ);
    m3_mul(SQ, S, SQS);
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            J[6 * i + j] = S[i][j];
            J[6 * i + j + 3] = -SQS[i][j];
            J[6 * (i + 3) + j] = 0.0;
            J[6 * (i + 3) + j + 3] = S[i][j];
        }
}

// ---- symmetric 3x3 eigen-decomposition (the plane fit of a voxel: kb_registration_constraints) ----------------------
// Cyclic Jacobi. A closed-form (trigonometric) solver loses its eigenvectors when eigenvalues nearly coincide, which is
// exactly what collinear and blob-like voxels produce; Jacobi rotations keep V orthonormal to a few ulps and resolve
// repeated and zero eigenvalues. One rotation (P, Q) zeroes a[P][Q] (Numerical Recipes' stable form, tau = s / (1 + c)).
template <int P, int Q>
KB_HD void sym3_rotate(double (&a)[3][3], double (&v)[3][3]) {
    constexpr int R = 3 - P - Q;
    const double apq = a[P][Q];
    if (apq == 0.0) return;
    const double theta = (a[Q][Q] - a[P][P]) / (2.0 * apq);
    double t = 1.0 / (fabs(theta) + sqrt(1.0 + theta * theta));  // theta^2 overflows -> t = 0: a[P][Q] is negligible
    if (theta < 0.0) t = -t;
    const double c = 1.0 / sqrt(t * t + 1.0), s = t * c, tau = s / (1.0 + c);
    a[P][P] -= t * apq;
    a[Q][Q] += t * apq;
    a[P][Q] = a[Q][P] = 0.0;
    const double arp = a[R][P], arq = a[R][Q];
    a[R][P] = a[P][R] = arp - s * (arq + tau * arp);
    a[R][Q] = a[Q][R] = arq + s * (arp - tau * arq);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double vp = v[k][P], vq = v[k][Q];
        v[k][P] = vp - s * (vq + tau * vp);
        v[k][Q] = vq + s * (vp - tau * vq);
    }
}

// c = the 6 unique entries (xx, xy, xz, yy, yz, zz). lam: eigenvalues ascending; vec[k] = unit eigenvector of lam[k].
// At most 16 sweeps (a 3x3 converges quadratically in 4-6); a sweep ends the loop when the off-diagonal part is below
// 1e-36 of the squared Frobenius norm, i.e. below rounding.
KB_HD void sym3_eig(const double c[6], double lam[3], V3 vec[3]) {
    double a[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
    double v[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
    for (int sweep = 0; sweep < 16; ++sweep) {
        const double off = (a[0][1] * a[0][1] + a[0][2] * a[0][2]) + a[1][2] * a[1][2];
        const double diag = (a[0][0] * a[0][0] + a[1][1] * a[1][1]) + a[2][2] * a[2][2];
        if (!(off > 1e-36 * (diag + 2.0 * off))) break;
        sym3_rotate<0, 1>(a, v);
        sym3_rotate<0, 2>(a, v);
        sym3_rotate<1, 2>(a, v);
    }
    double l[3] = {a[0][0], a[1][1], a[2][2]};
    int o[3] = {0, 1, 2};
    // three compare-exchanges (ascending, stable)
    if (l[o[1]] < l[o[0]]) { const int t = o[0]; o[0] = o[1]; o[1] = t; }
    if (l[o[2]] < l[o[1]]) { const int t = o[1]; o[1] = o[2]; o[2] = t; }
    if (l[o[1]] < l[o[0]]) { const int t = o[0]; o[0] = o[1]; o[1] = t; }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        // (selects instead of indexing with o[k]: the arrays stay in registers)
        const int j = o[k];
        lam[k] = j == 0 ? l[0] : (j == 1 ? l[1] : l[2]);
        vec[k] = j == 0 ? V3{v[0][0], v[1][0], v[2][0]} : (j == 1 ? V3{v[0][1], v[1][1], v[2][1]} : V3{v[0][2], v[1][2], v[2][2]});
    }
}

}  // namespace kb
