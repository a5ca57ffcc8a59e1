// FP64 manifold arithmetic of the 23-DOF FAST-LIO state, host+device.
//
// Follows the pieces of the reference's IKFoM / MTK toolkit that
// esekf::update_iterated_dyn_share_modified touches
// (include/IKFoM_toolkit/esekfom/esekfom.hpp:1619-1931):
//   state_ikfom layout        include/use-ikfom.hpp:12-21   (DOF 23, flat storage 26 doubles)
//   vect  boxplus/boxminus    mtk/types/vect.hpp:117-122
//   SO3   boxplus/boxminus    mtk/types/SOn.hpp:233-239, exp/log :284-297
//   S2    boxplus/boxminus, S2_Bx, S2_Nx_yy, S2_Mx   mtk/types/S2.hpp:136-281 (S2_typ = 1, length 9.809)
//   A_matrix, exp, log, cos_sinc_sqrt                 mtk/src/mtkmath.hpp:142-176, 235-288
// including their quirks (SURVEY.md traps T4, T5, T7).
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define FL_HD __host__ __device__ __forceinline__
#define FL_COLD __host__ __device__ __noinline__
#else
#define FL_HD inline
#define FL_COLD
#endif

namespace fl {

constexpr int NDOF = 23;
constexpr int XLEN = 26;
// flat state offsets
constexpr int X_POS = 0, X_ROT = 3, X_OFFR = 7, X_OFFT = 11, X_VEL = 14, X_BG = 17, X_BA = 20, X_GRAV = 23;
constexpr double S2_LEN = 98090.0 / 10000.0;     // use-ikfom.hpp:8
constexpr double MTK_TOL = 1e-11;                // MTK::tolerance<double>(), mtkmath.hpp:121

struct D3 { double x, y, z; };
struct Q4 { double x, y, z, w; };               // Eigen coeffs() order

FL_HD D3 d3(double x, double y, double z) { D3 r; r.x = x; r.y = y; r.z = z; return r; }
FL_HD D3 operator+(const D3& a, const D3& b) { return d3(a.x + b.x, a.y + b.y, a.z + b.z); }
FL_HD D3 operator-(const D3& a, const D3& b) { return d3(a.x - b.x, a.y - b.y, a.z - b.z); }
FL_HD D3 operator*(const D3& a, double s) { return d3(a.x * s, a.y * s, a.z * s); }
FL_HD double dot3(const D3& a, const D3& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
FL_HD D3 cross3(const D3& a, const D3& b) { return d3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
FL_HD double norm3(const D3& a) { return sqrt(dot3(a, a)); }

// 3x3 row-major
struct M33 { double m[9]; };
FL_HD M33 hat3(const D3& v) { M33 r = {{0, -v.z, v.y, v.z, 0, -v.x, -v.y, v.x, 0}}; return r; }
FL_HD M33 eye33() { M33 r = {{1, 0, 0, 0, 1, 0, 0, 0, 1}}; return r; }
FL_HD M33 mul33(const M33& a, const M33& b) {
    M33 r;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
        double s = 0; for (int k = 0; k < 3; k++) s += a.m[i * 3 + k] * b.m[k * 3 + j];
        r.m[i * 3 + j] = s;
    }
    return r;
}
FL_HD D3 mul33v(const M33& a, const D3& b) {
    return d3(a.m[0] * b.x + a.m[1] * b.y + a.m[2] * b.z, a.m[3] * b.x + a.m[4] * b.y + a.m[5] * b.z,
              a.m[6] * b.x + a.m[7] * b.y + a.m[8] * b.z);
}
FL_HD M33 transpose33(const M33& a) { M33 r = {{a.m[0], a.m[3], a.m[6], a.m[1], a.m[4], a.m[7], a.m[2], a.m[5], a.m[8]}}; return r; }

// Quaternion algebra with Eigen's formulas (Eigen/src/Geometry/Quaternion.h)
FL_HD Q4 qmul(const Q4& a, const Q4& b) {
    Q4 r;
    r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
    r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
    r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
    r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
    return r;
}
FL_HD Q4 qconj(const Q4& q) { Q4 r; r.x = -q.x; r.y = -q.y; r.z = -q.z; r.w = q.w; return r; }
FL_HD D3 qrot(const Q4& q, const D3& v) {           // QuaternionBase::_transformVector
    D3 qv = d3(q.x, q.y, q.z);
    D3 uv = cross3(qv, v);
    uv = uv + uv;
    return (v + uv * q.w) + cross3(qv, uv);
}
FL_HD M33 qmat(const Q4& q) {                       // QuaternionBase::toRotationMatrix
    const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
    const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
    const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
    const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
    M33 r = {{1 - (tyy + tzz), txy - twz, txz + twy, txy + twz, 1 - (txx + tzz), tyz - twx, txz - twy, tyz + twx, 1 - (txx + tyy)}};
    return r;
}

// mtkmath.hpp:142-176  (Taylor branch verbatim; the sqrt/cos/sin branch is out of line)
FL_COLD static void cos_sinc_exact(double x2, double& c, double& sinc) {
    double x = sqrt(x2);
    c = cos(x); sinc = sin(x) / x;
}
FL_HD void cos_sinc_sqrt(double x2, double& c, double& sinc) {
    const double taylor_n_bound = 1.220703125e-04;                   // sqrt(sqrt(eps<double>))
    if (x2 >= taylor_n_bound) { cos_sinc_exact(x2, c, sinc); return; }
    const double inv[7] = {1 / 3., 1 / 4., 1 / 5., 1 / 6., 1 / 7., 1 / 8., 1 / 9.};
    double cosi = 1., s = 1.;
    double term = -1 / 2. * x2;
    for (int i = 0; i < 3; ++i) {
        cosi += term;
        term *= inv[2 * i];
        s += term;
        term *= -inv[2 * i + 1] * x2;
    }
    c = cosi; sinc = s;
}
// mtkmath.hpp:249-256
FL_HD Q4 mtk_exp(const D3& v, double scale) {
    double c, sinc;
    cos_sinc_sqrt(scale * scale * dot3(v, v), c, sinc);
    double mult = sinc * scale;
    Q4 r; r.x = mult * v.x; r.y = mult * v.y; r.z = mult * v.z; r.w = c;
    return r;
}
FL_HD Q4 so3_exp(const D3& v) { return mtk_exp(v, 0.5); }            // SOn.hpp:284-288
// Exact forms (transcendental calls) are kept out of line: the filter only ever sees small
// tangent vectors, for which the series below are accurate to the last bits of FP64 and avoid
// hundreds of cold instructions in the single-block solve.
FL_COLD static D3 so3_log_exact(const Q4& q) {                       // SOn.hpp:293-297 -> mtkmath.hpp:268-288 (T7)
    D3 v = d3(q.x, q.y, q.z);
    double nv = norm3(v);
    if (nv < MTK_TOL) nv = MTK_TOL;
    double s = 2.0 / nv * atan(nv / q.w);
    return v * s;
}
FL_HD D3 so3_log(const Q4& q) {
    // 2 atan(nv / w) / nv = (2 / w) * atan(r) / r,  r = nv / w;  atan(r)/r = 1 - r^2/3 + r^4/5 - ...
    const double nv2 = q.x * q.x + q.y * q.y + q.z * q.z;
    const double r2 = nv2 / (q.w * q.w);
    if (!(r2 < 2.5e-3) || nv2 < MTK_TOL * MTK_TOL) return so3_log_exact(q);
    double p = 1.0 / 17.0;
    p = 1.0 / 15.0 - r2 * p; p = 1.0 / 13.0 - r2 * p; p = 1.0 / 11.0 - r2 * p; p = 1.0 / 9.0 - r2 * p;
    p = 1.0 / 7.0 - r2 * p;  p = 1.0 / 5.0 - r2 * p;  p = 1.0 / 3.0 - r2 * p;  p = 1.0 - r2 * p;
    return d3(q.x, q.y, q.z) * (2.0 / q.w * p);
}
FL_COLD static M33 A_matrix_exact(const D3& v) {                     // mtkmath.hpp:235-248
    double sq = v.x * v.x + v.y * v.y + v.z * v.z;
    double n = sqrt(sq);
    if (n < MTK_TOL) return eye33();
    M33 h = hat3(v), hh = mul33(h, h), r = eye33();
    double a = (1 - cos(n)) / sq, b = (1 - sin(n) / n) / sq;
    for (int i = 0; i < 9; i++) r.m[i] += a * h.m[i] + b * hh.m[i];
    return r;
}
FL_HD M33 A_matrix(const D3& v) {
    // (1 - cos n)/n^2 = 1/2 - n^2/24 + n^4/720 - ... ;  (1 - sin n / n)/n^2 = 1/6 - n^2/120 + n^4/5040 - ...
    const double sq = v.x * v.x + v.y * v.y + v.z * v.z;
    if (!(sq < 0.04)) return A_matrix_exact(v);
    if (sq < MTK_TOL * MTK_TOL) return eye33();
    double a = 1.0 / 87178291200.0;                       // 1/14!
    a = 1.0 / 479001600.0 - sq * a; a = 1.0 / 3628800.0 - sq * a; a = 1.0 / 40320.0 - sq * a;
    a = 1.0 / 720.0 - sq * a; a = 1.0 / 24.0 - sq * a; a = 0.5 - sq * a;
    double b = 1.0 / 1307674368000.0;                     // 1/15!
    b = 1.0 / 6227020800.0 - sq * b; b = 1.0 / 39916800.0 - sq * b; b = 1.0 / 362880.0 - sq * b;
    b = 1.0 / 5040.0 - sq * b; b = 1.0 / 120.0 - sq * b; b = 1.0 / 6.0 - sq * b;
    // hat(v)^2 = v v^T - |v|^2 I
    M33 r;
    r.m[0] = 1.0 + b * (v.x * v.x - sq); r.m[1] = -a * v.z + b * v.x * v.y;  r.m[2] = a * v.y + b * v.x * v.z;
    r.m[3] = a * v.z + b * v.x * v.y;    r.m[4] = 1.0 + b * (v.y * v.y - sq); r.m[5] = -a * v.x + b * v.y * v.z;
    r.m[6] = -a * v.y + b * v.x * v.z;   r.m[7] = a * v.x + b * v.y * v.z;   r.m[8] = 1.0 + b * (v.z * v.z - sq);
    return r;
}

// ---- S2, S2_typ == 1 (S2.hpp:214-239)
FL_HD void S2_Bx(const D3& v, double B[6]) {          // 3x2 row-major
    // S2.hpp:214-239 divides every entry by (L + v.x) and by L; here ONE reciprocal each (this runs in the single-warp solver,
    // where an FP64 division is ~40 dependent instructions) -- the entries stay within 3 ulps of max|B| of the reference's
    const double L = S2_LEN;
    constexpr double invL = 1.0 / S2_LEN;
    if (v.x + L > MTK_TOL) {
        const double r = 1.0 / (L + v.x);
        const double yy = v.y * v.y * r, zy = v.z * v.y * r, zz = v.z * v.z * r;
        B[0] = -v.y * invL;      B[1] = -v.z * invL;
        B[2] = (L - yy) * invL;  B[3] = -zy * invL;
        B[4] = -zy * invL;       B[5] = (L - zz) * invL;
    } else {
        for (int i = 0; i < 6; i++) B[i] = 0;
        B[3] = -1; B[4] = 1;
    }
}
FL_HD D3 S2_boxplus(const D3& v, double d0, double d1) {              // S2.hpp:136-142
    double B[6]; S2_Bx(v, B);
    D3 Bu = d3(B[0] * d0 + B[1] * d1, B[2] * d0 + B[3] * d1, B[4] * d0 + B[5] * d1);
    return mul33v(qmat(mtk_exp(Bu, 0.5)), v);
}
FL_COLD static double s2_theta_over_sin_exact(double v_sin2, double v_cos) {
    const double v_sin = sqrt(v_sin2);
    return atan2(v_sin, v_cos) / v_sin;
}
// `Bo` = S2_Bx(other): the update calls this with other = x_propagated.grav, fixed for the whole update
FL_HD void S2_boxminus_B(const D3& self, const D3& other, const double Bo[6], double& r0, double& r1) {   // S2.hpp:144-167
    const D3 cr = mul33v(hat3(self), other);
    const double v_sin2 = dot3(cr, cr);
    const double v_cos = dot3(self, other);
    if (v_sin2 < MTK_TOL * MTK_TOL) {
        // theta = atan2(v_sin, v_cos) is 0 for aligned and pi for opposed vectors
        if (v_cos < 0.0) { r0 = 3.1415926; r1 = 0; } else { r0 = 0; r1 = 0; }
        return;
    }
    // theta / v_sin = atan(t) / (t v_cos),  t = v_sin / v_cos
    double f;
    const double t2 = v_sin2 / (v_cos * v_cos);
    if (v_cos > 0.0 && t2 < 2.5e-3) {
        double p = 1.0 / 17.0;
        p = 1.0 / 15.0 - t2 * p; p = 1.0 / 13.0 - t2 * p; p = 1.0 / 11.0 - t2 * p; p = 1.0 / 9.0 - t2 * p;
        p = 1.0 / 7.0 - t2 * p;  p = 1.0 / 5.0 - t2 * p;  p = 1.0 / 3.0 - t2 * p;  p = 1.0 - t2 * p;
        f = p / v_cos;
    } else {
        f = s2_theta_over_sin_exact(v_sin2, v_cos);
    }
    const D3 hv = mul33v(hat3(other), self);
    r0 = f * (Bo[0] * hv.x + Bo[2] * hv.y + Bo[4] * hv.z);
    r1 = f * (Bo[1] * hv.x + Bo[3] * hv.y + Bo[5] * hv.z);
}
FL_HD void S2_boxminus(const D3& self, const D3& other, double& r0, double& r1) {
    double B[6]; S2_Bx(other, B);
    S2_boxminus_B(self, other, B, r0, r1);
}
FL_HD void S2_Nx_yy(const D3& v, double N[6]) {                       // 2x3, S2.hpp:262-267
    double B[6]; S2_Bx(v, B);
    M33 h = hat3(v);
    for (int i = 0; i < 2; i++) for (int j = 0; j < 3; j++) {
        double s = 0; for (int k = 0; k < 3; k++) s += B[k * 2 + i] * h.m[k * 3 + j];
        N[i * 3 + j] = 1 / S2_LEN / S2_LEN * s;
    }
}
// 3x2, S2.hpp:269-281.  T4: the reference's exp(.., scalar(1/2)) has scale 0 (integer division) -- the identity rotation: the
// product with it is dropped here (E h == h exactly).  `B` = S2_Bx(v).
FL_HD void S2_Mx_B(const D3& v, const double B[6], double d0, double d1, double M[6]) {
    M33 h = hat3(v);
    M33 T = h;
    if (!(sqrt(d0 * d0 + d1 * d1) < MTK_TOL)) {
        D3 Bu = d3(B[0] * d0 + B[1] * d1, B[2] * d0 + B[3] * d1, B[4] * d0 + B[5] * d1);
        T = mul33(h, transpose33(A_matrix(Bu)));
    }
    for (int i = 0; i < 3; i++) for (int j = 0; j < 2; j++) {
        double s = 0; for (int k = 0; k < 3; k++) s += T.m[i * 3 + k] * B[k * 2 + j];
        M[i * 2 + j] = -s;
    }
}
FL_HD void S2_Mx(const D3& v, double d0, double d1, double M[6]) {
    double B[6]; S2_Bx(v, B);
    S2_Mx_B(v, B, d0, d1, M);
}
// 2x2 = Nx(x.grav) * Mx(x_prop.grav, delta)      (esekfom.hpp:1686-1690);  `Bp` = S2_Bx(grav_prop)
FL_HD void S2_congruence_B(const D3& grav_now, const D3& grav_prop, const double Bp[6], double d0, double d1, double M2[4]) {
    double N[6], Mx[6];
    S2_Nx_yy(grav_now, N);
    S2_Mx_B(grav_prop, Bp, d0, d1, Mx);
    for (int i = 0; i < 2; i++) for (int j = 0; j < 2; j++) {
        double s = 0; for (int k = 0; k < 3; k++) s += N[i * 3 + k] * Mx[k * 2 + j];
        M2[i * 2 + j] = s;
    }
}
FL_HD void S2_congruence(const D3& grav_now, const D3& grav_prop, double d0, double d1, double M2[4]) {
    double B[6]; S2_Bx(grav_prop, B);
    S2_congruence_B(grav_now, grav_prop, B, d0, d1, M2);
}

// ---- compound state (build_manifold.hpp:192-200)
FL_HD Q4 ldq(const double* p) { Q4 q; q.x = p[0]; q.y = p[1]; q.z = p[2]; q.w = p[3]; return q; }
FL_HD D3 ld3(const double* p) { return d3(p[0], p[1], p[2]); }
FL_HD void stq(double* p, const Q4& q) { p[0] = q.x; p[1] = q.y; p[2] = q.z; p[3] = q.w; }
FL_HD void st3(double* p, const D3& v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; }

FL_HD void state_boxplus(double* x, const double* d) {
    for (int i = 0; i < 3; i++) { x[X_POS + i] += d[i]; x[X_OFFT + i] += d[9 + i]; x[X_VEL + i] += d[12 + i]; x[X_BG + i] += d[15 + i]; x[X_BA + i] += d[18 + i]; }
    stq(x + X_ROT, qmul(ldq(x + X_ROT), so3_exp(d3(d[3], d[4], d[5]))));
    stq(x + X_OFFR, qmul(ldq(x + X_OFFR), so3_exp(d3(d[6], d[7], d[8]))));
    st3(x + X_GRAV, S2_boxplus(ld3(x + X_GRAV), d[21], d[22]));
}
// r = a [-] b
FL_HD void state_boxminus(const double* a, const double* b, double* r) {
    for (int i = 0; i < 3; i++) { r[i] = a[X_POS + i] - b[X_POS + i]; r[9 + i] = a[X_OFFT + i] - b[X_OFFT + i]; r[12 + i] = a[X_VEL + i] - b[X_VEL + i]; r[15 + i] = a[X_BG + i] - b[X_BG + i]; r[18 + i] = a[X_BA + i] - b[X_BA + i]; }
    D3 l1 = so3_log(qmul(qconj(ldq(b + X_ROT)), ldq(a + X_ROT)));
    D3 l2 = so3_log(qmul(qconj(ldq(b + X_OFFR)), ldq(a + X_OFFR)));
    st3(r + 3, l1); st3(r + 6, l2);
    S2_boxminus(ld3(a + X_GRAV), ld3(b + X_GRAV), r[21], r[22]);
}

}  // namespace fl
