// The plane term of a rig calibration's correspondence in the sensor's own tangent, shared by k_calib (calib.cu) and
// k_calib_clock (calib_clock.cu). Like frame.cuh it is compiled inside the including module's own namespace (the module
// defines kb to its name around the include).
#pragma once

#include "frame.cuh"

namespace kb {

// the plane term of one correspondence (map point m of sensor point p, nearest map point q) for this lane's value, as
// plane_term (frame.cuh) forms it, but with the voxel normal rotated into the sensor frame: n_s = (R_k R_j)^T n and
// J = [n_s, p x n_s], the sensor tangent of the right perturbation E_j Exp(dx)
__device__ __forceinline__ double calib_plane_term(const MapView &m, const V3 &mp, const V3 &q, const V3 &p,
                                                   const Q4 &to_sensor, int lane, int ji, int jj) {
    const int3 v = point_to_voxel(q.x, q.y, q.z, m.vdiv);
    int cnt = 0;
    const int slot = map_find(m, v.x, v.y, v.z, &cnt);
    if (slot < 0 || cnt < 3) return 0.0;
    const double *blk = m.points + static_cast<size_t>(slot) * m.cap * 3;
    double sx = 0.0, sy = 0.0, sz = 0.0;
    for (int k = lane; k < cnt; k += 32) {
        sx += blk[3 * k];
        sy += blk[3 * k + 1];
        sz += blk[3 * k + 2];
    }
    const double inv_m = 1.0 / static_cast<double>(cnt);
    const V3 mu{warp_sum(sx) * inv_m, warp_sum(sy) * inv_m, warp_sum(sz) * inv_m};
    double c[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int k = lane; k < cnt; k += 32) {
        const V3 d = V3{blk[3 * k], blk[3 * k + 1], blk[3 * k + 2]} - mu;
        c[0] += d.x * d.x;
        c[1] += d.x * d.y;
        c[2] += d.x * d.z;
        c[3] += d.y * d.y;
        c[4] += d.y * d.z;
        c[5] += d.z * d.z;
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) c[i] = warp_sum(c[i]) * inv_m;
    double lam[3];
    V3 ev[3];
    sym3_eig(c, lam, ev);
    const double a = lam[2] > 0.0 ? (lam[1] - lam[0]) / lam[2] : 0.0;
    const V3 n = ev[0];
    const V3 r = mp - q;
    const double e = (n.x * r.x + n.y * r.y) + n.z * r.z;
    const V3 ns = q_rotate(to_sensor, n);
    const V3 pn = cross(p, ns);
    const double J[6] = {ns.x, ns.y, ns.z, pn.x, pn.y, pn.z};
    double Ji = 0.0, Jj = 0.0;
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        Ji = (ji == i) ? J[i] : Ji;
        Jj = (jj == i) ? J[i] : Jj;
    }
    if (lane == 0) return 1.0;
    if (lane == 1) return a;
    if (lane == 2) return a * (e * e);
    return a * (Ji * Jj);
}

}  // namespace kb
