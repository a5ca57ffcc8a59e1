// ============================================================================
// ORACLE -- TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the
// product path; only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs may load this library.
//
// CPU restatement (plain C++14, no Eigen / Boost / PCL / ROS -- none of them
// exist in this container) of FAST-LIO2's per-scan iterated-EKF measurement
// update.  Every function cites the reference file:line it follows
// (paths relative to /root/reference).
//
//   h_share_model                         src/laserMapping.cpp:638-754
//   esti_plane<float>                     include/common_lib.h:225-257
//   update_iterated_dyn_share_modified    include/IKFoM_toolkit/esekfom/esekfom.hpp:1619-1931
//   MTK SO3 / S2 / vect boxplus, boxminus include/IKFoM_toolkit/mtk/types/{SOn,S2,vect}.hpp
//   A_matrix, exp, log, cos_sinc_sqrt     include/IKFoM_toolkit/mtk/src/mtkmath.hpp
//   state_ikfom layout                    include/use-ikfom.hpp:6-21
//
// Third-party arithmetic that the reference pulls from an ABSENT dependency
// (Eigen >= 3.3.4, unpinned: README.md:74, CMakeLists.txt:59) is restated
// from Eigen 3.3's published algorithms:
//   * ColPivHouseholderQR<Matrix<float,5,3>>::solve   (used at common_lib.h:241)
//   * Matrix<double,23,23>::inverse() = PartialPivLU   (esekfom.hpp:1782,1802)
//   * Quaternion * Vector3, Quaternion * Quaternion, toRotationMatrix()
//
// PARITY STATUS: the reference ships no tests, fixtures or golden vectors for
// this path (SURVEY.md section 4) => "parity unpinned" by the reference.  The
// kNN half is pinned against the reference's own unmodified ikd_Tree.cpp
// compiled into oracle/_ref (see oracle/Makefile); the EKF half is pinned only
// by self-consistency properties (tests/test_oracle_*.py).
// ============================================================================
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <limits>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

constexpr int NUM_MATCH_POINTS = 5;   // common_lib.h:26
constexpr int N_DOF = 23;             // state_ikfom::DOF (use-ikfom.hpp:12-21)
constexpr int X_LEN = 26;             // flat state: pos3 rot4 offR4 offT3 vel3 bg3 ba3 grav3
constexpr double S2_LENGTH = 98090.0 / 10000.0;  // use-ikfom.hpp:8  S2<double,98090,10000,1>
constexpr double TOL_D = 1e-11;       // MTK::tolerance<double>()  mtkmath.hpp:121

// ---------------------------------------------------------------- tiny linalg
struct V3 { double v[3]; double& operator[](int i){return v[i];} double operator[](int i) const {return v[i];} };
struct M3 { double m[3][3]; };
struct Quat { double x, y, z, w; };   // Eigen coeffs() order (x,y,z,w)

inline V3 v3(double a, double b, double c) { return V3{{a, b, c}}; }
inline V3 add(const V3& a, const V3& b) { return v3(a[0]+b[0], a[1]+b[1], a[2]+b[2]); }
inline V3 sub(const V3& a, const V3& b) { return v3(a[0]-b[0], a[1]-b[1], a[2]-b[2]); }
inline V3 scale(const V3& a, double s) { return v3(a[0]*s, a[1]*s, a[2]*s); }
inline double dot(const V3& a, const V3& b) { return a[0]*b[0] + a[1]*b[1] + a[2]*b[2]; }
inline V3 cross(const V3& a, const V3& b) {
    return v3(a[1]*b[2]-a[2]*b[1], a[2]*b[0]-a[0]*b[2], a[0]*b[1]-a[1]*b[0]);
}
inline double norm(const V3& a) { return std::sqrt(dot(a, a)); }

inline M3 hat(const V3& v) {  // mtkmath.hpp:178-185
    M3 r = {{{0, -v[2], v[1]}, {v[2], 0, -v[0]}, {-v[1], v[0], 0}}};
    return r;
}
inline M3 eye3() { M3 r = {{{1,0,0},{0,1,0},{0,0,1}}}; return r; }
inline M3 mul(const M3& a, const M3& b) {
    M3 r;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) {
        double s = 0; for (int k = 0; k < 3; k++) s += a.m[i][k] * b.m[k][j];
        r.m[i][j] = s;
    }
    return r;
}
inline V3 mul(const M3& a, const V3& b) {
    return v3(a.m[0][0]*b[0]+a.m[0][1]*b[1]+a.m[0][2]*b[2],
              a.m[1][0]*b[0]+a.m[1][1]*b[1]+a.m[1][2]*b[2],
              a.m[2][0]*b[0]+a.m[2][1]*b[1]+a.m[2][2]*b[2]);
}
inline M3 transpose(const M3& a) {
    M3 r; for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r.m[i][j] = a.m[j][i]; return r;
}

// Eigen::Quaternion product (Eigen/src/Geometry/Quaternion.h quat_product)
inline Quat qmul(const Quat& a, const Quat& b) {
    Quat r;
    r.w = a.w*b.w - a.x*b.x - a.y*b.y - a.z*b.z;
    r.x = a.w*b.x + a.x*b.w + a.y*b.z - a.z*b.y;
    r.y = a.w*b.y + a.y*b.w + a.z*b.x - a.x*b.z;
    r.z = a.w*b.z + a.z*b.w + a.x*b.y - a.y*b.x;
    return r;
}
inline Quat qconj(const Quat& q) { return Quat{-q.x, -q.y, -q.z, q.w}; }
// Eigen QuaternionBase::_transformVector
inline V3 qrot(const Quat& q, const V3& v) {
    V3 qv = v3(q.x, q.y, q.z);
    V3 uv = cross(qv, v);
    uv = add(uv, uv);
    return add(add(v, scale(uv, q.w)), cross(qv, uv));
}
// Eigen QuaternionBase::toRotationMatrix
inline M3 qmat(const Quat& q) {
    const double tx = 2*q.x, ty = 2*q.y, tz = 2*q.z;
    const double twx = tx*q.w, twy = ty*q.w, twz = tz*q.w;
    const double txx = tx*q.x, txy = ty*q.x, txz = tz*q.x;
    const double tyy = ty*q.y, tyz = tz*q.y, tzz = tz*q.z;
    M3 r;
    r.m[0][0] = 1-(tyy+tzz); r.m[0][1] = txy-twz;     r.m[0][2] = txz+twy;
    r.m[1][0] = txy+twz;     r.m[1][1] = 1-(txx+tzz); r.m[1][2] = tyz-twx;
    r.m[2][0] = txz-twy;     r.m[2][1] = tyz+twx;     r.m[2][2] = 1-(txx+tyy);
    return r;
}

// ------------------------------------------------------------ MTK math pieces
// mtkmath.hpp:142-176  cos_sinc_sqrt<double>
inline void cos_sinc_sqrt(double x2, double& c, double& sinc) {
    static const double taylor_0_bound = std::numeric_limits<double>::epsilon();
    static const double taylor_2_bound = std::sqrt(taylor_0_bound);
    static const double taylor_n_bound = std::sqrt(taylor_2_bound);
    if (x2 >= taylor_n_bound) {
        double x = std::sqrt(x2);
        c = std::cos(x); sinc = std::sin(x) / x;
        return;
    }
    static const double inv[] = {1/3., 1/4., 1/5., 1/6., 1/7., 1/8., 1/9.};
    double cosi = 1., s = 1.;
    double term = -1/2. * x2;
    for (int i = 0; i < 3; ++i) {
        cosi += term;
        term *= inv[2*i];
        s += term;
        term *= -inv[2*i+1] * x2;
    }
    c = cosi; sinc = s;
}

// mtkmath.hpp:249-256  exp<scalar,3>(result, vec, scale) -> returns w
inline Quat mtk_exp(const V3& vec, double scl) {
    double norm2 = dot(vec, vec);
    double c, sinc;
    cos_sinc_sqrt(scl * scl * norm2, c, sinc);
    double mult = sinc * scl;
    return Quat{mult * vec[0], mult * vec[1], mult * vec[2], c};
}
// SOn.hpp:284-288  SO3::exp(dvec, scale=1): w = exp(vec, dvec, scale/2)
inline Quat so3_exp(const V3& d) { return mtk_exp(d, 0.5); }

// mtkmath.hpp:268-288 log<scalar,3>(result, w, vec, scale, plus_minus_periodicity)
// called from SOn.hpp:293-297 with scale=2, periodicity=true
inline V3 so3_log(const Quat& q) {
    V3 vec = v3(q.x, q.y, q.z);
    double nv = norm(vec);
    if (nv < TOL_D) nv = TOL_D;     // periodicity==true: the w<0 branch is skipped
    double s = 2.0 / nv * std::atan(nv / q.w);
    return scale(vec, s);
}

// mtkmath.hpp:235-248  A_matrix
inline M3 A_matrix(const V3& v) {
    double squaredNorm = v[0]*v[0] + v[1]*v[1] + v[2]*v[2];
    double nrm = std::sqrt(squaredNorm);
    if (nrm < TOL_D) return eye3();
    M3 h = hat(v), hh = mul(h, h), r = eye3();
    double a = (1 - std::cos(nrm)) / squaredNorm;
    double b = (1 - std::sin(nrm) / nrm) / squaredNorm;
    for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r.m[i][j] += a * h.m[i][j] + b * hh.m[i][j];
    return r;
}

// ------------------------------------------------------------------- S2 (typ 1)
// S2.hpp:179-240, S2_typ == 1 branch (use-ikfom.hpp:8)
inline void S2_Bx(const V3& vec, double res[3][2]) {
    const double L = S2_LENGTH;
    if (vec[0] + L > TOL_D) {
        res[0][0] = -vec[1];                          res[0][1] = -vec[2];
        res[1][0] = L - vec[1]*vec[1]/(L+vec[0]);     res[1][1] = -vec[2]*vec[1]/(L+vec[0]);
        res[2][0] = -vec[2]*vec[1]/(L+vec[0]);        res[2][1] = L - vec[2]*vec[2]/(L+vec[0]);
        for (int i = 0; i < 3; i++) for (int j = 0; j < 2; j++) res[i][j] /= L;
    } else {
        for (int i = 0; i < 3; i++) for (int j = 0; j < 2; j++) res[i][j] = 0;
        res[1][1] = -1; res[2][0] = 1;
    }
}
// S2.hpp:136-142 boxplus
inline V3 S2_boxplus(const V3& vec, const double delta[2]) {
    double Bx[3][2]; S2_Bx(vec, Bx);
    V3 Bu = v3(Bx[0][0]*delta[0]+Bx[0][1]*delta[1], Bx[1][0]*delta[0]+Bx[1][1]*delta[1], Bx[2][0]*delta[0]+Bx[2][1]*delta[1]);
    Quat r = mtk_exp(Bu, 0.5);
    return mul(qmat(r), vec);
}
// S2.hpp:144-167 boxminus : res = this [-] other
inline void S2_boxminus(const V3& self, const V3& other, double res[2]) {
    double v_sin = norm(mul(hat(self), other));
    double v_cos = dot(self, other);
    double theta = std::atan2(v_sin, v_cos);
    if (v_sin < TOL_D) {
        if (std::fabs(theta) > TOL_D) { res[0] = 3.1415926; res[1] = 0; }
        else { res[0] = 0; res[1] = 0; }
    } else {
        double Bx[3][2]; S2_Bx(other, Bx);
        V3 hv = mul(hat(other), self);
        double f = theta / v_sin;
        for (int j = 0; j < 2; j++) res[j] = f * (Bx[0][j]*hv[0] + Bx[1][j]*hv[1] + Bx[2][j]*hv[2]);
    }
}
// S2.hpp:262-267  S2_Nx_yy : res(2x3) = 1/L/L * Bx^T * hat(vec)
inline void S2_Nx_yy(const V3& vec, double res[2][3]) {
    double Bx[3][2]; S2_Bx(vec, Bx);
    M3 h = hat(vec);
    for (int i = 0; i < 2; i++) for (int j = 0; j < 3; j++) {
        double s = 0; for (int k = 0; k < 3; k++) s += Bx[k][i] * h.m[k][j];
        res[i][j] = 1 / S2_LENGTH / S2_LENGTH * s;
    }
}
// S2.hpp:269-281 S2_Mx. NOTE trap T4: scalar(1/2) is integer division == 0, so
// exp_delta is the identity rotation (S2.hpp:277).
inline void S2_Mx(const V3& vec, const double delta[2], double res[3][2]) {
    double Bx[3][2]; S2_Bx(vec, Bx);
    M3 h = hat(vec);
    double dn = std::sqrt(delta[0]*delta[0] + delta[1]*delta[1]);
    if (dn < TOL_D) {
        for (int i = 0; i < 3; i++) for (int j = 0; j < 2; j++) {
            double s = 0; for (int k = 0; k < 3; k++) s += h.m[i][k] * Bx[k][j];
            res[i][j] = -s;
        }
    } else {
        V3 Bu = v3(Bx[0][0]*delta[0]+Bx[0][1]*delta[1], Bx[1][0]*delta[0]+Bx[1][1]*delta[1], Bx[2][0]*delta[0]+Bx[2][1]*delta[1]);
        Quat ed = mtk_exp(Bu, double(1/2));          // == identity (T4)
        M3 E = qmat(ed);
        M3 At = transpose(A_matrix(Bu));
        M3 T = mul(mul(E, h), At);
        for (int i = 0; i < 3; i++) for (int j = 0; j < 2; j++) {
            double s = 0; for (int k = 0; k < 3; k++) s += T.m[i][k] * Bx[k][j];
            res[i][j] = -s;
        }
    }
}

// --------------------------------------------------------------------- state
struct State {            // use-ikfom.hpp:12-21
    V3 pos; Quat rot; Quat offR; V3 offT; V3 vel; V3 bg; V3 ba; V3 grav;
};
inline State load_state(const double* x) {
    State s;
    s.pos = v3(x[0], x[1], x[2]);
    s.rot = Quat{x[3], x[4], x[5], x[6]};
    s.offR = Quat{x[7], x[8], x[9], x[10]};
    s.offT = v3(x[11], x[12], x[13]);
    s.vel = v3(x[14], x[15], x[16]);
    s.bg = v3(x[17], x[18], x[19]);
    s.ba = v3(x[20], x[21], x[22]);
    s.grav = v3(x[23], x[24], x[25]);
    return s;
}
inline void store_state(const State& s, double* x) {
    for (int i = 0; i < 3; i++) { x[i] = s.pos[i]; x[11+i] = s.offT[i]; x[14+i] = s.vel[i]; x[17+i] = s.bg[i]; x[20+i] = s.ba[i]; x[23+i] = s.grav[i]; }
    x[3] = s.rot.x; x[4] = s.rot.y; x[5] = s.rot.z; x[6] = s.rot.w;
    x[7] = s.offR.x; x[8] = s.offR.y; x[9] = s.offR.z; x[10] = s.offR.w;
}
// build_manifold.hpp:192-194 boxplus, DOF order: pos0 rot3 offR6 offT9 vel12 bg15 ba18 grav21
inline void state_boxplus(State& s, const double* d) {
    for (int i = 0; i < 3; i++) { s.pos[i] += d[i]; s.offT[i] += d[9+i]; s.vel[i] += d[12+i]; s.bg[i] += d[15+i]; s.ba[i] += d[18+i]; }  // vect.hpp:117-119
    s.rot = qmul(s.rot, so3_exp(v3(d[3], d[4], d[5])));      // SOn.hpp:233-236
    s.offR = qmul(s.offR, so3_exp(v3(d[6], d[7], d[8])));
    double dg[2] = {d[21], d[22]};
    s.grav = S2_boxplus(s.grav, dg);
}
// build_manifold.hpp:198-200 boxminus: res = a [-] b
inline void state_boxminus(const State& a, const State& b, double* r) {
    for (int i = 0; i < 3; i++) { r[i] = a.pos[i]-b.pos[i]; r[9+i] = a.offT[i]-b.offT[i]; r[12+i] = a.vel[i]-b.vel[i]; r[15+i] = a.bg[i]-b.bg[i]; r[18+i] = a.ba[i]-b.ba[i]; }
    V3 l1 = so3_log(qmul(qconj(b.rot), a.rot));              // SOn.hpp:237-239
    V3 l2 = so3_log(qmul(qconj(b.offR), a.offR));
    for (int i = 0; i < 3; i++) { r[3+i] = l1[i]; r[6+i] = l2[i]; }
    double g[2]; S2_boxminus(a.grav, b.grav, g);
    r[21] = g[0]; r[22] = g[1];
}

// ---------------------------------------- dense NxN inverse (Eigen PartialPivLU)
// Restates Matrix::inverse() for n > 4: PartialPivLU (row pivoting on the largest
// |a_ik|, unblocked for n<=... ) followed by solving for the identity.
static bool inverse_lu(const double* A, double* Ainv, int n) {
    std::vector<double> lu(A, A + n * n);
    std::vector<int> perm(n);
    for (int i = 0; i < n; i++) perm[i] = i;
    for (int k = 0; k < n; k++) {
        int piv = k; double best = std::fabs(lu[k*n+k]);
        for (int i = k+1; i < n; i++) { double a = std::fabs(lu[i*n+k]); if (a > best) { best = a; piv = i; } }
        if (best == 0.0) return false;
        if (piv != k) { for (int j = 0; j < n; j++) std::swap(lu[k*n+j], lu[piv*n+j]); std::swap(perm[k], perm[piv]); }
        double d = lu[k*n+k];
        for (int i = k+1; i < n; i++) lu[i*n+k] /= d;
        for (int i = k+1; i < n; i++) { double f = lu[i*n+k]; if (f != 0.0) for (int j = k+1; j < n; j++) lu[i*n+j] -= f * lu[k*n+j]; }
    }
    for (int c = 0; c < n; c++) {
        std::vector<double> y(n);
        for (int i = 0; i < n; i++) {
            double s = (perm[i] == c) ? 1.0 : 0.0;
            for (int j = 0; j < i; j++) s -= lu[i*n+j] * y[j];
            y[i] = s;
        }
        for (int i = n-1; i >= 0; i--) {
            double s = y[i];
            for (int j = i+1; j < n; j++) s -= lu[i*n+j] * Ainv[j*n+c];
            Ainv[i*n+c] = s / lu[i*n+i];
        }
    }
    return true;
}

// ------------------------------------------------ esti_plane (common_lib.h:225-257)
// float 5x3 least squares A x = -1 via Eigen 3.3 ColPivHouseholderQR
// (Eigen/src/QR/ColPivHouseholderQR.h computeInPlace + _solve_impl,
//  Eigen/src/Householder/Householder.h makeHouseholder / applyHouseholderOnTheLeft).
// Branches taken, for the tests: transp, nonzero_pivots, tiny_tail[k] (makeHouseholder's tailSq <= min branch) and
// norm[k][j] for j > k: 0 not visited (j <= k), 1 downdated, 2 recomputed, 3 skipped (normsUpdated[j] == 0).
struct PlaneTrace { int nonzero_pivots; int transp[3]; int tiny_tail[3]; int norm[3][3]; };

static bool esti_plane_f(float pca_result[4], const float pts[NUM_MATCH_POINTS][3], float threshold, PlaneTrace* trace = nullptr) {
    if (trace) memset(trace, 0, sizeof(*trace));
    const int rows = NUM_MATCH_POINTS, cols = 3, size = 3;
    float qr[5][3];
    float c[5];
    for (int j = 0; j < rows; j++) { qr[j][0] = pts[j][0]; qr[j][1] = pts[j][1]; qr[j][2] = pts[j][2]; c[j] = -1.0f; }
    float hCoeffs[3];
    int transp[3];
    float normsUpdated[3], normsDirect[3];
    for (int k = 0; k < cols; k++) {
        float s = 0.f; for (int i = 0; i < rows; i++) s += qr[i][k] * qr[i][k];
        normsDirect[k] = std::sqrt(s); normsUpdated[k] = normsDirect[k];
    }
    const float eps = std::numeric_limits<float>::epsilon();
    float maxn = std::max(normsUpdated[0], std::max(normsUpdated[1], normsUpdated[2]));
    const float threshold_helper = (maxn * eps) * (maxn * eps) / float(rows);
    const float norm_downdate_threshold = std::sqrt(eps);
    int nonzero_pivots = size;
    float maxpivot = 0.f;
    for (int k = 0; k < size; k++) {
        int biggest = k; float bn = normsUpdated[k];
        for (int j = k+1; j < cols; j++) if (normsUpdated[j] > bn) { bn = normsUpdated[j]; biggest = j; }
        float biggest_sq = bn * bn;
        if (nonzero_pivots == size && biggest_sq < threshold_helper * float(rows - k)) nonzero_pivots = k;
        transp[k] = biggest;
        if (k != biggest) {
            for (int i = 0; i < rows; i++) std::swap(qr[i][k], qr[i][biggest]);
            std::swap(normsUpdated[k], normsUpdated[biggest]);
            std::swap(normsDirect[k], normsDirect[biggest]);
        }
        // makeHouseholderInPlace on qr.col(k).tail(rows-k)
        float tailSq = 0.f; for (int i = k+1; i < rows; i++) tailSq += qr[i][k] * qr[i][k];
        float c0 = qr[k][k];
        float tau, beta;
        const float tol = (std::numeric_limits<float>::min)();
        if (trace) trace->tiny_tail[k] = tailSq <= tol;
        if (tailSq <= tol) {
            tau = 0.f; beta = c0;
            for (int i = k+1; i < rows; i++) qr[i][k] = 0.f;
        } else {
            beta = std::sqrt(c0 * c0 + tailSq);
            if (c0 >= 0.f) beta = -beta;
            for (int i = k+1; i < rows; i++) qr[i][k] = qr[i][k] / (c0 - beta);
            tau = (beta - c0) / beta;
        }
        hCoeffs[k] = tau;
        qr[k][k] = beta;
        if (std::fabs(beta) > maxpivot) maxpivot = std::fabs(beta);
        // apply H_k to the trailing columns
        if (tau != 0.f) {
            for (int j = k+1; j < cols; j++) {
                float tmp = 0.f;
                for (int i = k+1; i < rows; i++) tmp += qr[i][k] * qr[i][j];
                tmp += qr[k][j];
                qr[k][j] -= tau * tmp;
                for (int i = k+1; i < rows; i++) qr[i][j] -= tau * qr[i][k] * tmp;
            }
        }
        // column-norm downdate (LAPACK working note 176 style, as in Eigen 3.3)
        for (int j = k+1; j < cols; j++) {
            if (trace) trace->norm[k][j] = 3;
            if (normsUpdated[j] != 0.f) {
                float temp = std::fabs(qr[k][j]) / normsUpdated[j];
                temp = (1.f + temp) * (1.f - temp);
                temp = temp < 0.f ? 0.f : temp;
                float r = normsUpdated[j] / normsDirect[j];
                float temp2 = temp * r * r;
                if (trace) trace->norm[k][j] = temp2 <= norm_downdate_threshold ? 2 : 1;
                if (temp2 <= norm_downdate_threshold) {
                    float s = 0.f; for (int i = k+1; i < rows; i++) s += qr[i][j] * qr[i][j];
                    normsDirect[j] = std::sqrt(s);
                    normsUpdated[j] = normsDirect[j];
                } else {
                    normsUpdated[j] *= std::sqrt(temp);
                }
            }
        }
    }
    if (trace) { trace->nonzero_pivots = nonzero_pivots; for (int k = 0; k < 3; k++) trace->transp[k] = transp[k]; }
    // _solve_impl: c = Q^T b (first nonzero_pivots reflectors), back-substitute, un-permute
    for (int k = 0; k < nonzero_pivots; k++) {
        float tau = hCoeffs[k];
        if (tau != 0.f) {
            float tmp = 0.f;
            for (int i = k+1; i < rows; i++) tmp += qr[i][k] * c[i];
            tmp += c[k];
            c[k] -= tau * tmp;
            for (int i = k+1; i < rows; i++) c[i] -= tau * qr[i][k] * tmp;
        }
    }
    for (int i = nonzero_pivots - 1; i >= 0; i--) {
        float s = c[i];
        for (int j = i+1; j < nonzero_pivots; j++) s -= qr[i][j] * c[j];
        c[i] = s / qr[i][i];
    }
    // colsPermutation = product of transpositions; dst.row(perm[i]) = c[i]
    int perm[3] = {0, 1, 2};
    // PermutationMatrix built as: setIdentity; for k: applyTranspositionOnTheRight(k, transp[k])
    for (int k = 0; k < size; k++) std::swap(perm[k], perm[transp[k]]);
    float x[3] = {0.f, 0.f, 0.f};
    for (int i = 0; i < nonzero_pivots; i++) x[perm[i]] = c[i];
    // common_lib.h:243-256
    float n = std::sqrt(x[0]*x[0] + x[1]*x[1] + x[2]*x[2]);
    pca_result[0] = x[0] / n;
    pca_result[1] = x[1] / n;
    pca_result[2] = x[2] / n;
    pca_result[3] = float(1.0 / n);
    for (int j = 0; j < NUM_MATCH_POINTS; j++) {
        if (std::fabs(pca_result[0]*pts[j][0] + pca_result[1]*pts[j][1] + pca_result[2]*pts[j][2] + pca_result[3]) > threshold)
            return false;
    }
    return true;
}

// laserMapping.cpp:656-661
inline V3 body_to_world(const State& s, const float* pb, float pw[3]) {
    V3 p_global = add(qrot(s.rot, add(qrot(s.offR, v3(pb[0], pb[1], pb[2])), s.offT)), s.pos);
    pw[0] = float(p_global[0]); pw[1] = float(p_global[1]); pw[2] = float(p_global[2]);
    return p_global;
}

// laserMapping.cpp:671
inline bool knn_gate(int cnt, float d2_last) { return cnt < NUM_MATCH_POINTS ? false : (d2_last > 5 ? false : true); }

// laserMapping.cpp:680-681: returns the score; pd2 out
inline float plane_score(const float pabcd[4], const float pw[3], const float* pb, float& pd2) {
    V3 p_body = v3(pb[0], pb[1], pb[2]);
    pd2 = pabcd[0] * pw[0] + pabcd[1] * pw[1] + pabcd[2] * pw[2] + pabcd[3];          // :680
    return float(1 - 0.9 * std::fabs(pd2) / std::sqrt(norm(p_body)));                // :681 (T8)
}

// laserMapping.cpp:723-751: one row of h_x and its entry of h, from normvec = (n, pd2)
inline void jacobian_row(const State& s, const float* pb, const float* nv, int extrinsic_est_en, double* row, double& h) {
    V3 point_this_be = v3(pb[0], pb[1], pb[2]);
    M3 point_be_crossmat = hat(point_this_be);
    V3 point_this = add(qrot(s.offR, point_this_be), s.offT);
    M3 point_crossmat = hat(point_this);
    V3 norm_vec = v3(nv[0], nv[1], nv[2]);
    V3 C = qrot(qconj(s.rot), norm_vec);
    V3 A = mul(point_crossmat, C);
    row[0] = norm_vec[0]; row[1] = norm_vec[1]; row[2] = norm_vec[2];
    row[3] = A[0]; row[4] = A[1]; row[5] = A[2];
    if (extrinsic_est_en) {
        // point_be_crossmat * s.offset_R_L_I.conjugate() * C : Eigen evaluates
        // (Matrix3 * Quaternion) by converting the quaternion to a rotation matrix.
        V3 B = mul(mul(point_be_crossmat, qmat(qconj(s.offR))), C);
        row[6] = B[0]; row[7] = B[1]; row[8] = B[2];
        row[9] = C[0]; row[10] = C[1]; row[11] = C[2];
    }
    h = -double(nv[3]);                                                              // :751
}

}  // namespace

// ============================================================================
// C interface (ctypes).  kNN is injected so that the SAME restatement can run
// on top of (a) the reference's own unmodified ikd-Tree (oracle/_ref), or
// (b) the port in oracle/knn_port.cpp.
// ============================================================================
extern "C" {

// Returns the number of neighbours found (<= k).  out_pts: k x 4 floats
// (x,y,z,intensity), ascending by distance; out_d2: k floats.
typedef int (*oracle_knn_fn)(void* ctx, const float* q_xyz, int k, float* out_pts4, float* out_d2);

struct OraclePassLog {
    int searched;        // 1 if this pass ran the kNN (ekfom_data.converge on entry)
    int valid;           // dyn_share.valid after h_share_model
    int effct;           // effct_feat_num
    int converged;       // dyn_share.converge after the step
    double res_sum;      // total_residual
    double HtH[144];     // h_x^T h_x (12x12 row-major)
    double Hth[12];      // h_x^T h
    double x_after[26];  // state after boxplus
};

int oracle_esti_plane(const float* pts15, float threshold, float* out4) {
    float p[5][3];
    for (int i = 0; i < 5; i++) for (int j = 0; j < 3; j++) p[i][j] = pts15[i*3+j];
    return esti_plane_f(out4, p, threshold) ? 1 : 0;
}

// oracle_esti_plane plus the branches it took: trace16 = nonzero_pivots, transp[3], tiny_tail[3], norm[3][3] (PlaneTrace)
int oracle_esti_plane_trace(const float* pts15, float threshold, float* out4, int* trace16) {
    static_assert(sizeof(PlaneTrace) == 16 * sizeof(int), "PlaneTrace layout");
    float p[5][3];
    for (int i = 0; i < 5; i++) for (int j = 0; j < 3; j++) p[i][j] = pts15[i*3+j];
    PlaneTrace tr;
    const int ok = esti_plane_f(out4, p, threshold, &tr) ? 1 : 0;
    memcpy(trace16, &tr, sizeof(tr));
    return ok;
}

// One point of h_share_model (laserMapping.cpp:656-692, :723-751) with every stage evaluated whatever the gates before it
// decided: pw[3]; flags[3] = kNN gate (:671), plane fit accepted (:678), score gate (:683); pabcd[4]; pd2; score; row[12]
// (zero beyond 6 without extrinsic estimation); h.  out25 = pw, flags, pabcd, pd2, score, row, h as doubles.
void oracle_measure_point(const double* x26, const float* pb3, const float* near15, int cnt, float d2_last, int extrinsic_est_en,
                          double* out25) {
    const State s = load_state(x26);
    float pw[3];
    body_to_world(s, pb3, pw);
    const bool gate = knn_gate(cnt, d2_last);
    float pn[5][3];
    for (int i = 0; i < 5; i++) for (int j = 0; j < 3; j++) pn[i][j] = near15[i*3+j];
    float pabcd[4];
    const bool ok = esti_plane_f(pabcd, pn, 0.1f);
    float pd2;
    const float sc = plane_score(pabcd, pw, pb3, pd2);
    const float nv[4] = {pabcd[0], pabcd[1], pabcd[2], pd2};
    double row[12] = {0}, h;
    jacobian_row(s, pb3, nv, extrinsic_est_en, row, h);
    double* o = out25;
    for (int i = 0; i < 3; i++) *o++ = pw[i];
    *o++ = gate; *o++ = ok; *o++ = sc > 0.9;
    for (int i = 0; i < 4; i++) *o++ = pabcd[i];
    *o++ = pd2; *o++ = sc;
    for (int i = 0; i < 12; i++) *o++ = row[i];
    *o++ = h;
}

void oracle_state_boxplus(double* x26, const double* d23) { State s = load_state(x26); state_boxplus(s, d23); store_state(s, x26); }
void oracle_state_boxminus(const double* a26, const double* b26, double* r23) { state_boxminus(load_state(a26), load_state(b26), r23); }
int oracle_inverse(const double* A, double* Ainv, int n) { return inverse_lu(A, Ainv, n) ? 0 : -1; }
void oracle_A_matrix(const double* v3in, double* out9) { M3 a = A_matrix(v3(v3in[0], v3in[1], v3in[2])); memcpy(out9, a.m, sizeof(a.m)); }
// The MTK pieces one at a time (row-major outputs), for the manifold tests of the device code
void oracle_so3_exp(const double* v3in, double* q4) { Quat q = so3_exp(v3(v3in[0], v3in[1], v3in[2])); q4[0] = q.x; q4[1] = q.y; q4[2] = q.z; q4[3] = q.w; }
void oracle_so3_log(const double* q4, double* out3) { V3 l = so3_log(Quat{q4[0], q4[1], q4[2], q4[3]}); for (int i = 0; i < 3; i++) out3[i] = l[i]; }
void oracle_S2_Bx(const double* v3in, double* out6) { double b[3][2]; S2_Bx(v3(v3in[0], v3in[1], v3in[2]), b); memcpy(out6, b, sizeof(b)); }
void oracle_S2_boxminus(const double* self_other6, double* out2) {
    S2_boxminus(v3(self_other6[0], self_other6[1], self_other6[2]), v3(self_other6[3], self_other6[4], self_other6[5]), out2);
}
void oracle_S2_Nx_yy(const double* v3in, double* out6) { double n[2][3]; S2_Nx_yy(v3(v3in[0], v3in[1], v3in[2]), n); memcpy(out6, n, sizeof(n)); }
void oracle_S2_Mx(const double* v3_delta2, double* out6) {
    double m[3][2]; S2_Mx(v3(v3_delta2[0], v3_delta2[1], v3_delta2[2]), v3_delta2 + 3, m); memcpy(out6, m, sizeof(m));
}
void oracle_transform_point(const double* x26, const float* pb, float* pw) {
    body_to_world(load_state(x26), pb, pw);
}

// ----------------------------------------------------------------------------
// One full update_iterated_dyn_share_modified call (esekfom.hpp:1619-1931)
// with h_share_model (laserMapping.cpp:638-754) inlined as the measurement
// callback.  Dynamic sizes: the reference's static 100000-point arrays
// (laserMapping.cpp:76,94,112-114) are lifted.
//
//  body_pts   Q x 4 float (x,y,z,intensity)       feats_down_body
//  x26        in/out flat state                   kf.x_
//  P          in/out 23x23 row-major              kf.P_
//  nearest    out Q x 5 x 4 float, nearest_cnt out Q   (Nearest_Points after the last search pass)
//  selected   out Q bytes (point_selected_surf after the last pass)
//  logs       out, capacity max_iter+1 entries; n_passes out
// Returns 0.
// ----------------------------------------------------------------------------
int oracle_update_iterated(const float* body_pts, int Q, double* x26, double* P,
                           int maximum_iter, double R, const double* limit23, int extrinsic_est_en,
                           oracle_knn_fn knn, void* knn_ctx, int nthreads,
                           float* nearest, int* nearest_cnt, unsigned char* selected_out,
                           OraclePassLog* logs, int* n_passes) {
    const int n = N_DOF;
    State x_ = load_state(x26);
    std::vector<double> P_(P, P + n*n), L_(n*n);
    // per-scan persistent arrays (globals in laserMapping.cpp:76,94,102,112)
    std::vector<unsigned char> point_selected_surf(Q, 0);
    std::vector<float> res_last(Q, 0.f);
    std::vector<float> normvec(size_t(Q) * 4, 0.f);           // (n, pd2)
    std::vector<float> Nearest(size_t(Q) * 20, 0.f);
    std::vector<int> NearestCnt(Q, 0);
    std::vector<float> world(size_t(Q) * 3, 0.f);

    // esekfom.hpp:1621-1631
    bool valid = true, converge = true;
    int t = 0;
    const State x_propagated = x_;
    const std::vector<double> P_propagated = P_;
    int dof_Measurement = 0;
    double K_h[N_DOF];
    std::vector<double> K_x(n*n, 0.0);
    double dx_new[N_DOF];
    for (int i = 0; i < n; i++) dx_new[i] = 0;
    int pass = 0;
    if (n_passes) *n_passes = 0;
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#endif

    std::vector<double> h_x;   // effct x 12
    std::vector<double> h;     // effct

    for (int it = -1; it < maximum_iter; it++, pass++) {   // esekfom.hpp:1633
        valid = true;
        OraclePassLog* log = logs ? &logs[pass] : nullptr;
        if (log) { memset(log, 0, sizeof(*log)); log->searched = converge ? 1 : 0; }
        // ================= h_share_model (laserMapping.cpp:638-754) =================
        const State s = x_;
        double total_residual = 0.0;
        const bool do_search = converge;
#pragma omp parallel for schedule(static)
        for (int i = 0; i < Q; i++) {                                   // :650
            const float* pb = &body_pts[size_t(i) * 4];
            float pw[3];
            body_to_world(s, pb, pw);                                     // :657
            world[size_t(i)*3+0] = pw[0]; world[size_t(i)*3+1] = pw[1]; world[size_t(i)*3+2] = pw[2];
            float* near = &Nearest[size_t(i) * 20];
            if (do_search) {                                              // :667-672
                float d2[NUM_MATCH_POINTS];
                float tmp[NUM_MATCH_POINTS * 4];
                int cnt = knn(knn_ctx, pw, NUM_MATCH_POINTS, tmp, d2);
                NearestCnt[i] = cnt;
                for (int j = 0; j < cnt * 4; j++) near[j] = tmp[j];
                point_selected_surf[i] = knn_gate(cnt, d2[NUM_MATCH_POINTS - 1]) ? 1 : 0;
            }
            if (!point_selected_surf[i]) continue;                        // :674
            point_selected_surf[i] = 0;                                   // :677
            float pabcd[4];
            float pn[NUM_MATCH_POINTS][3];
            for (int j = 0; j < NUM_MATCH_POINTS; j++) { pn[j][0] = near[j*4]; pn[j][1] = near[j*4+1]; pn[j][2] = near[j*4+2]; }
            if (esti_plane_f(pabcd, pn, 0.1f)) {                          // :678
                float pd2;
                const float sc = plane_score(pabcd, pw, pb, pd2);         // :680-681
                if (sc > 0.9) {                                           // :683
                    point_selected_surf[i] = 1;
                    normvec[size_t(i)*4+0] = pabcd[0]; normvec[size_t(i)*4+1] = pabcd[1];
                    normvec[size_t(i)*4+2] = pabcd[2]; normvec[size_t(i)*4+3] = pd2;
                    res_last[i] = std::fabs(pd2);
                }
            }
        }
        // compaction :695-706
        std::vector<int> eff; eff.reserve(Q);
        for (int i = 0; i < Q; i++) if (point_selected_surf[i]) { eff.push_back(i); total_residual += res_last[i]; }
        const int effct_feat_num = int(eff.size());
        if (log) { log->effct = effct_feat_num; log->res_sum = total_residual; }
        if (effct_feat_num < 1) {                                         // :708-713
            valid = false;
        } else {
            h_x.assign(size_t(effct_feat_num) * 12, 0.0);                 // :720
            h.assign(effct_feat_num, 0.0);
            for (int r = 0; r < effct_feat_num; r++) {                    // :723-752
                const int i = eff[r];
                jacobian_row(s, &body_pts[size_t(i) * 4], &normvec[size_t(i) * 4], extrinsic_est_en, &h_x[size_t(r) * 12], h[r]);
            }
        }
        if (log) log->valid = valid ? 1 : 0;
        // ============================ back in esekfom.hpp ============================
        if (!valid) { if (log) { log->converged = converge ? 1 : 0; store_state(x_, log->x_after); } continue; }   // :1638-1641
        dof_Measurement = effct_feat_num;                                  // :1650
        double dx[N_DOF];
        state_boxminus(x_, x_propagated, dx);                              // :1652
        for (int i = 0; i < n; i++) dx_new[i] = dx[i];
        P_ = P_propagated;                                                 // :1657
        // SO3 blocks, idx 3 (rot) then 6 (offset_R_L_I)  :1659-1676
        const int so3_idx[2] = {3, 6};
        for (int b = 0; b < 2; b++) {
            int idx = so3_idx[b];
            M3 J = transpose(A_matrix(v3(dx[idx], dx[idx+1], dx[idx+2])));   // T5
            V3 seg = mul(J, v3(dx_new[idx], dx_new[idx+1], dx_new[idx+2]));
            for (int i = 0; i < 3; i++) dx_new[idx+i] = seg[i];
            for (int i = 0; i < n; i++) {
                V3 col = mul(J, v3(P_[(idx)*n+i], P_[(idx+1)*n+i], P_[(idx+2)*n+i]));
                for (int k = 0; k < 3; k++) P_[(idx+k)*n+i] = col[k];
            }
            for (int i = 0; i < n; i++) {
                V3 rw = v3(P_[i*n+idx], P_[i*n+idx+1], P_[i*n+idx+2]);
                // row(1x3) * J^T  ==  (J * row^T)^T
                V3 out = mul(J, rw);
                for (int k = 0; k < 3; k++) P_[i*n+idx+k] = out[k];
            }
        }
        // S2 block idx 21  :1678-1699
        {
            const int idx = 21;
            double seg[2] = {dx[idx], dx[idx+1]};
            double Nx[2][3], Mx[3][2], M[2][2];
            S2_Nx_yy(x_.grav, Nx);
            S2_Mx(x_propagated.grav, seg, Mx);
            for (int i = 0; i < 2; i++) for (int j = 0; j < 2; j++) { double sacc = 0; for (int k = 0; k < 3; k++) sacc += Nx[i][k] * Mx[k][j]; M[i][j] = sacc; }
            double d0 = M[0][0]*dx_new[idx] + M[0][1]*dx_new[idx+1];
            double d1 = M[1][0]*dx_new[idx] + M[1][1]*dx_new[idx+1];
            dx_new[idx] = d0; dx_new[idx+1] = d1;
            for (int i = 0; i < n; i++) {
                double a = P_[idx*n+i], bq = P_[(idx+1)*n+i];
                P_[idx*n+i] = M[0][0]*a + M[0][1]*bq; P_[(idx+1)*n+i] = M[1][0]*a + M[1][1]*bq;
            }
            for (int i = 0; i < n; i++) {
                double a = P_[i*n+idx], bq = P_[i*n+idx+1];
                P_[i*n+idx] = a*M[0][0] + bq*M[0][1]; P_[i*n+idx+1] = a*M[1][0] + bq*M[1][1];
            }
        }
        // Normal equations (for the log + the large-m branch)
        double HTH[144], HTh[12];
        for (int a = 0; a < 12; a++) { for (int b = 0; b < 12; b++) HTH[a*12+b] = 0; HTh[a] = 0; }
        for (int r = 0; r < dof_Measurement; r++) {
            const double* row = &h_x[size_t(r) * 12];
            for (int a = 0; a < 12; a++) { for (int b = 0; b < 12; b++) HTH[a*12+b] += row[a] * row[b]; HTh[a] += row[a] * h[r]; }
        }
        if (log) { memcpy(log->HtH, HTH, sizeof(HTH)); memcpy(log->Hth, HTh, sizeof(HTh)); }
        if (n > dof_Measurement) {                                        // :1715-1744 (T6)
            const int m = dof_Measurement;
            std::vector<double> Hc(size_t(m) * n, 0.0);
            for (int r = 0; r < m; r++) for (int a = 0; a < 12; a++) Hc[r*n+a] = h_x[size_t(r)*12+a];
            std::vector<double> PHt(size_t(n) * m, 0.0), S(size_t(m) * m, 0.0), Sinv(size_t(m) * m, 0.0);
            for (int i = 0; i < n; i++) for (int r = 0; r < m; r++) { double sacc = 0; for (int k = 0; k < n; k++) sacc += P_[i*n+k] * Hc[r*n+k]; PHt[i*m+r] = sacc; }
            for (int r = 0; r < m; r++) for (int c2 = 0; c2 < m; c2++) { double sacc = 0; for (int k = 0; k < n; k++) sacc += Hc[r*n+k] * PHt[k*m+c2]; S[r*m+c2] = sacc / R + (r == c2 ? 1.0 : 0.0); }
            inverse_lu(S.data(), Sinv.data(), m);
            std::vector<double> K(size_t(n) * m, 0.0);
            for (int i = 0; i < n; i++) for (int c2 = 0; c2 < m; c2++) { double sacc = 0; for (int k = 0; k < m; k++) sacc += PHt[i*m+k] * Sinv[k*m+c2]; K[i*m+c2] = sacc / R; }
            for (int i = 0; i < n; i++) { double sacc = 0; for (int r = 0; r < m; r++) sacc += K[i*m+r] * h[r]; K_h[i] = sacc; }
            for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) { double sacc = 0; for (int r = 0; r < m; r++) sacc += K[i*m+r] * Hc[r*n+j]; K_x[i*n+j] = sacc; }
        } else {                                                          // :1782-1809
            std::vector<double> PR(n*n), P_temp(n*n), P_inv(n*n);
            for (int i = 0; i < n*n; i++) PR[i] = P_[i] / R;
            inverse_lu(PR.data(), P_temp.data(), n);
            for (int a = 0; a < 12; a++) for (int b = 0; b < 12; b++) P_temp[a*n+b] += HTH[a*12+b];
            inverse_lu(P_temp.data(), P_inv.data(), n);
            for (int i = 0; i < n; i++) { double sacc = 0; for (int a = 0; a < 12; a++) sacc += P_inv[i*n+a] * HTh[a]; K_h[i] = sacc; }
            std::fill(K_x.begin(), K_x.end(), 0.0);
            for (int i = 0; i < n; i++) for (int b = 0; b < 12; b++) { double sacc = 0; for (int a = 0; a < 12; a++) sacc += P_inv[i*n+a] * HTH[a*12+b]; K_x[i*n+b] = sacc; }
        }
        // :1815-1817
        double dx_[N_DOF];
        for (int i = 0; i < n; i++) {
            double sacc = K_h[i];
            for (int j = 0; j < n; j++) sacc += (K_x[i*n+j] - (i == j ? 1.0 : 0.0)) * dx_new[j];
            dx_[i] = sacc;
        }
        state_boxplus(x_, dx_);
        converge = true;                                                   // :1818-1827
        for (int i = 0; i < n; i++) if (std::fabs(dx_[i]) > limit23[i]) { converge = false; break; }
        if (converge) t++;
        if (!t && it == maximum_iter - 2) converge = true;                 // :1829-1832 (T2)
        if (log) { log->converged = converge ? 1 : 0; store_state(x_, log->x_after); }
        if (t > 1 || it == maximum_iter - 1) {                             // :1834
            L_ = P_;
            for (int b = 0; b < 2; b++) {                                  // :1838-1863
                int idx = so3_idx[b];
                M3 J = transpose(A_matrix(v3(dx_[idx], dx_[idx+1], dx_[idx+2])));
                for (int i = 0; i < n; i++) {
                    V3 col = mul(J, v3(P_[idx*n+i], P_[(idx+1)*n+i], P_[(idx+2)*n+i]));
                    for (int k = 0; k < 3; k++) L_[(idx+k)*n+i] = col[k];
                }
                for (int i = 0; i < 12; i++) {
                    V3 col = mul(J, v3(K_x[idx*n+i], K_x[(idx+1)*n+i], K_x[(idx+2)*n+i]));
                    for (int k = 0; k < 3; k++) K_x[(idx+k)*n+i] = col[k];
                }
                for (int i = 0; i < n; i++) {
                    V3 lr = mul(J, v3(L_[i*n+idx], L_[i*n+idx+1], L_[i*n+idx+2]));
                    V3 pr = mul(J, v3(P_[i*n+idx], P_[i*n+idx+1], P_[i*n+idx+2]));
                    for (int k = 0; k < 3; k++) { L_[i*n+idx+k] = lr[k]; P_[i*n+idx+k] = pr[k]; }
                }
            }
            {                                                              // :1865-1900
                const int idx = 21;
                double seg[2] = {dx_[idx], dx_[idx+1]};
                double Nx[2][3], Mx[3][2], M[2][2];
                S2_Nx_yy(x_.grav, Nx);
                S2_Mx(x_propagated.grav, seg, Mx);
                for (int i = 0; i < 2; i++) for (int j = 0; j < 2; j++) { double sacc = 0; for (int k = 0; k < 3; k++) sacc += Nx[i][k] * Mx[k][j]; M[i][j] = sacc; }
                for (int i = 0; i < n; i++) {
                    double a = P_[idx*n+i], bq = P_[(idx+1)*n+i];
                    L_[idx*n+i] = M[0][0]*a + M[0][1]*bq; L_[(idx+1)*n+i] = M[1][0]*a + M[1][1]*bq;
                }
                for (int i = 0; i < 12; i++) {
                    double a = K_x[idx*n+i], bq = K_x[(idx+1)*n+i];
                    K_x[idx*n+i] = M[0][0]*a + M[0][1]*bq; K_x[(idx+1)*n+i] = M[1][0]*a + M[1][1]*bq;
                }
                for (int i = 0; i < n; i++) {
                    double a = L_[i*n+idx], bq = L_[i*n+idx+1];
                    L_[i*n+idx] = a*M[0][0] + bq*M[0][1]; L_[i*n+idx+1] = a*M[1][0] + bq*M[1][1];
                    double pa = P_[i*n+idx], pb2 = P_[i*n+idx+1];
                    P_[i*n+idx] = pa*M[0][0] + pb2*M[0][1]; P_[i*n+idx+1] = pa*M[1][0] + pb2*M[1][1];
                }
            }
            // P_ = L_ - K_x[:, :12] * P_[:12, :]   :1924
            std::vector<double> Pn(n*n);
            for (int i = 0; i < n; i++) for (int j = 0; j < n; j++) {
                double sacc = 0; for (int a = 0; a < 12; a++) sacc += K_x[i*n+a] * P_[a*n+j];
                Pn[i*n+j] = L_[i*n+j] - sacc;
            }
            P_ = Pn;
            pass++;
            break;
        }
    }
    if (n_passes) *n_passes = pass;
    store_state(x_, x26);
    memcpy(P, P_.data(), sizeof(double) * n * n);
    if (nearest) memcpy(nearest, Nearest.data(), sizeof(float) * size_t(Q) * 20);
    if (nearest_cnt) memcpy(nearest_cnt, NearestCnt.data(), sizeof(int) * Q);
    if (selected_out) memcpy(selected_out, point_selected_surf.data(), Q);
    return 0;
}

int oracle_pass_log_size() { return int(sizeof(OraclePassLog)); }

}  // extern "C"
