// The per-point measurement model of h_share_model (reference src/laserMapping.cpp:656-692, :723-751), host+device.
//
// Each function is what the update kernels run for one scan point: the body->world transform, the kNN gate, the 5-point
// plane fit (esti_plane, include/common_lib.h:225-257), the point-to-plane residual with its score gate, and one row of
// the measurement Jacobian.  They are FL_HD so that a test can run the same code on the host.
#pragma once
#include "common.cuh"
#include "lie.cuh"

namespace fl {

// ============================================================================= esti_plane
// float32 least squares A n = -1 on the 5 neighbours, column-pivoted Householder QR -- the
// algorithm the reference gets from Eigen (common_lib.h:241, colPivHouseholderQr().solve) --
// followed by the reference's normalisation and 0.1 m point-to-plane check (common_lib.h:243-256).
FL_HD bool esti_plane_dev(float pabcd[4], const float (&pt)[KNN_K][3], float threshold) {
    constexpr int rows = KNN_K, cols = 3, size = 3;
    float qr[rows][cols];
    float c[rows];
#pragma unroll
    for (int j = 0; j < rows; j++) { qr[j][0] = pt[j][0]; qr[j][1] = pt[j][1]; qr[j][2] = pt[j][2]; c[j] = -1.0f; }
    float hc[size];
    int transp[size];
    float nu[cols], nd[cols];
#pragma unroll
    for (int k = 0; k < cols; k++) {
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < rows; i++) s += qr[i][k] * qr[i][k];
        nd[k] = sqrtf(s); nu[k] = nd[k];
    }
    const float eps = 1.1920929e-07f;
    const float maxn = fmaxf(nu[0], fmaxf(nu[1], nu[2]));
    const float threshold_helper = (maxn * eps) * (maxn * eps) / float(rows);
    const float norm_downdate_threshold = sqrtf(eps);
    int nonzero_pivots = size;
#pragma unroll
    for (int k = 0; k < size; k++) {
        int biggest = k; float bn = nu[k];
#pragma unroll
        for (int j = k + 1; j < cols; j++) if (nu[j] > bn) { bn = nu[j]; biggest = j; }
        if (nonzero_pivots == size && bn * bn < threshold_helper * float(rows - k)) nonzero_pivots = k;
        transp[k] = biggest;
        if (k != biggest) {
#pragma unroll
            for (int j = k + 1; j < cols; j++) {
                if (j == biggest) {
#pragma unroll
                    for (int i = 0; i < rows; i++) { float t = qr[i][k]; qr[i][k] = qr[i][j]; qr[i][j] = t; }
                    float t = nu[k]; nu[k] = nu[j]; nu[j] = t;
                    t = nd[k]; nd[k] = nd[j]; nd[j] = t;
                }
            }
        }
        float tailSq = 0.f;
#pragma unroll
        for (int i = k + 1; i < rows; i++) tailSq += qr[i][k] * qr[i][k];
        const float c0 = qr[k][k];
        float tau, beta;
        if (tailSq <= 1.17549435e-38f) {
            tau = 0.f; beta = c0;
#pragma unroll
            for (int i = k + 1; i < rows; i++) qr[i][k] = 0.f;
        } else {
            beta = sqrtf(c0 * c0 + tailSq);
            if (c0 >= 0.f) beta = -beta;
#pragma unroll
            for (int i = k + 1; i < rows; i++) qr[i][k] = qr[i][k] / (c0 - beta);
            tau = (beta - c0) / beta;
        }
        hc[k] = tau;
        qr[k][k] = beta;
        if (tau != 0.f) {
#pragma unroll
            for (int j = k + 1; j < cols; j++) {
                float tmp = 0.f;
#pragma unroll
                for (int i = k + 1; i < rows; i++) tmp += qr[i][k] * qr[i][j];
                tmp += qr[k][j];
                qr[k][j] -= tau * tmp;
#pragma unroll
                for (int i = k + 1; i < rows; i++) qr[i][j] -= tau * qr[i][k] * tmp;
            }
        }
#pragma unroll
        for (int j = k + 1; j < cols; j++) {
            if (nu[j] != 0.f) {
                float temp = fabsf(qr[k][j]) / nu[j];
                temp = (1.f + temp) * (1.f - temp);
                temp = temp < 0.f ? 0.f : temp;
                const float r = nu[j] / nd[j];
                const float temp2 = temp * r * r;
                if (temp2 <= norm_downdate_threshold) {
                    float s = 0.f;
#pragma unroll
                    for (int i = k + 1; i < rows; i++) s += qr[i][j] * qr[i][j];
                    nd[j] = sqrtf(s); nu[j] = nd[j];
                } else {
                    nu[j] *= sqrtf(temp);
                }
            }
        }
    }
#pragma unroll
    for (int k = 0; k < size; k++) {
        if (k < nonzero_pivots) {
            const float tau = hc[k];
            if (tau != 0.f) {
                float tmp = 0.f;
#pragma unroll
                for (int i = k + 1; i < rows; i++) tmp += qr[i][k] * c[i];
                tmp += c[k];
                c[k] -= tau * tmp;
#pragma unroll
                for (int i = k + 1; i < rows; i++) c[i] -= tau * qr[i][k] * tmp;
            }
        }
    }
#pragma unroll
    for (int i = size - 1; i >= 0; i--) {
        if (i < nonzero_pivots) {
            float s = c[i];
#pragma unroll
            for (int j = i + 1; j < size; j++) if (j < nonzero_pivots) s -= qr[i][j] * c[j];
            c[i] = s / qr[i][i];
        }
    }
    int perm[3] = {0, 1, 2};
#pragma unroll
    for (int k = 0; k < size; k++) {
        // swap(perm[k], perm[transp[k]]) with static indexing
#pragma unroll
        for (int j = 0; j < size; j++) if (j == transp[k] && j != k) { int t = perm[k]; perm[k] = perm[j]; perm[j] = t; }
    }
    float x[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < size; i++) {
        if (i < nonzero_pivots) {
#pragma unroll
            for (int j = 0; j < 3; j++) if (perm[i] == j) x[j] = c[i];
        }
    }
    const float n = sqrtf(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    pabcd[0] = x[0] / n; pabcd[1] = x[1] / n; pabcd[2] = x[2] / n;
    pabcd[3] = (float)(1.0 / (double)n);
    bool ok = true;
#pragma unroll
    for (int j = 0; j < rows; j++)
        if (fabsf(pabcd[0] * pt[j][0] + pabcd[1] * pt[j][1] + pabcd[2] * pt[j][2] + pabcd[3]) > threshold) ok = false;
    return ok;
}

// ============================================================================= measurement model
struct PoseS {            // the part of the state h_share_model reads
    Q4 rot, offR; D3 pos, offT;
};
FL_HD PoseS load_pose(const double* x) {
    PoseS p; p.rot = ldq(x + X_ROT); p.offR = ldq(x + X_OFFR); p.pos = ld3(x + X_POS); p.offT = ld3(x + X_OFFT);
    return p;
}
// laserMapping.cpp:656-661; returns p_this = R_LI p_b + t_LI, which is also the lever arm of the Jacobian (:733)
FL_HD D3 body_to_world(const PoseS& s, const float4& pb, float& wx, float& wy, float& wz) {
    const D3 p_this = qrot(s.offR, d3(pb.x, pb.y, pb.z)) + s.offT;
    const D3 g = qrot(s.rot, p_this) + s.pos;
    wx = (float)g.x; wy = (float)g.y; wz = (float)g.z;
    return p_this;
}
// laserMapping.cpp:671: five neighbours found, the farthest within sqrt(5) m (a NaN distance passes, as in the reference)
FL_HD bool knn_gate(int cnt, float d2_last) { return cnt >= KNN_K && !(d2_last > 5.0f); }
// laserMapping.cpp:680: the point-to-plane residual of the world point
FL_HD float plane_residual(const float pabcd[4], float wx, float wy, float wz) {
    return pabcd[0] * wx + pabcd[1] * wy + pabcd[2] * wz + pabcd[3];
}
// laserMapping.cpp:681-683: the score gate, with srange = sqrt(|p_body|) (T8: the reference divides by the square root of
// the range).  Kept apart from plane_residual so that k_update can compute pd2 before it reads or caches srange: the
// other order schedules its instructions differently.
FL_HD bool score_gate(float pd2, double srange, float& score) {
    score = (float)(1 - 0.9 * fabs((double)pd2) / srange);
    return (double)score > 0.9;
}
// laserMapping.cpp:723-751: one row of h_x (12 wide) and the entry of h
template <bool EXTR>
FL_HD void jacobian_row(const PoseS& s, const float4& pb, const float4& nv, double* h, double& z) {
    D3 p_be = d3(pb.x, pb.y, pb.z);
    D3 p_this = qrot(s.offR, p_be) + s.offT;
    D3 n = d3(nv.x, nv.y, nv.z);
    D3 C = qrot(qconj(s.rot), n);
    D3 A = mul33v(hat3(p_this), C);
    h[0] = n.x; h[1] = n.y; h[2] = n.z; h[3] = A.x; h[4] = A.y; h[5] = A.z;
    if (EXTR) {
        D3 B = mul33v(mul33(hat3(p_be), qmat(qconj(s.offR))), C);
        h[6] = B.x; h[7] = B.y; h[8] = B.z; h[9] = C.x; h[10] = C.y; h[11] = C.z;
    }
    z = -(double)nv.w;
}

// the same with p_this = R_LI p_b + t_LI already at hand (body_to_world computes it on the way)
template <bool EXTR>
FL_HD void jacobian_row_at(const PoseS& s, const float4& pb, const D3& p_this, const float4& nv, double* h, double& z) {
    D3 n = d3(nv.x, nv.y, nv.z);
    D3 C = qrot(qconj(s.rot), n);
    D3 A = mul33v(hat3(p_this), C);
    h[0] = n.x; h[1] = n.y; h[2] = n.z; h[3] = A.x; h[4] = A.y; h[5] = A.z;
    if (EXTR) {
        D3 B = mul33v(mul33(hat3(d3(pb.x, pb.y, pb.z)), qmat(qconj(s.offR))), C);
        h[6] = B.x; h[7] = B.y; h[8] = B.z; h[9] = C.x; h[10] = C.y; h[11] = C.z;
    }
    z = -(double)nv.w;
}

}  // namespace fl
