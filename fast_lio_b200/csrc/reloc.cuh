// The grid of relocalisation hypotheses around a prior (fl_reloc_expand_grid_device), host+device: k_reloc_expand runs it on
// the device, and tests compile it for the host to check the numpy restatement against the very formula the kernel runs.
#pragma once
#include "../../include/fastlio_b200.h"
#include "lie.cuh"

namespace fl {

// The offset of grid index i on an axis of n points `step` apart, centred on the prior.
FL_HD double reloc_offset(int i, int n, double step) { return ((double)i - (double)(n - 1) / 2.0) * step; }

// Component c of hypothesis h, h = ((i_yaw n2 + i_z) n1 + i_y) n0 + i_x: pos + the world-frame offset, rot turned by the yaw
// offset about u = -grav / |grav| of the prior (rot = q_yaw * rot_prior), every other component the prior's.
FL_HD double reloc_component(const double* prior, const fl_reloc_grid_t& g, long long h, int c) {
    const int ix = (int)(h % g.n[0]);
    const int iy = (int)((h / g.n[0]) % g.n[1]);
    const int iz = (int)((h / ((long long)g.n[0] * g.n[1])) % g.n[2]);
    const int iw = (int)(h / ((long long)g.n[0] * g.n[1] * g.n[2]));
    if (c < X_ROT) {
        const int i = c == 0 ? ix : (c == 1 ? iy : iz);
        return prior[c] + reloc_offset(i, g.n[c], g.step[c]);
    }
    if (c >= X_ROT + 4) return prior[c];
    const double gx = prior[X_GRAV], gy = prior[X_GRAV + 1], gz = prior[X_GRAV + 2];
    const double gn = sqrt(gx * gx + gy * gy + gz * gz);
    const double half = 0.5 * reloc_offset(iw, g.n[3], g.step[3]);
    const double s = sin(half);
    Q4 qy;
    qy.x = -gx / gn * s; qy.y = -gy / gn * s; qy.z = -gz / gn * s; qy.w = cos(half);
    const Q4 r = qmul(qy, ldq(prior + X_ROT));
    return c == X_ROT ? r.x : (c == X_ROT + 1 ? r.y : (c == X_ROT + 2 ? r.z : r.w));
}

}  // namespace fl
