// The terms of the pose graph's cost that the host (kb_pose_graph_prior_chi2 in api_pose_graph.cu) and the device
// (pose_graph_edges.cuh) evaluate alike: the robust loss, and a prior's residual and Jacobian. Included inside the
// namespace of each unit that uses them, after se3.cuh.

// rho(s) and w = rho'(s): the Cauchy loss c^2 log(1 + s / c^2) for c > 0, the squared loss s for c = 0
KB_HD void robust_loss(double s, double c, double *rho, double *w) {
    if (c > 0.0) {
        const double c2 = c * c;
        *rho = c2 * log1p(s / c2);
        *w = 1.0 / (1.0 + s / c2);
    } else {
        *rho = s;
        *w = 1.0;
    }
}

enum { PG_POSE_PRIOR = 0, PG_POSITION_PRIOR = 1 };

// The residual r of a prior at the node's pose T, and s = r^T Omega r (Om: 6x6 row-major; a position prior's 3x3 in its
// top-left corner, zeros elsewhere).
//   pose prior, meas = Z^-1 as q(4) t(3):        r = Log(Z^-1 T)
//   position prior, meas = p(3), lever arm l(3): r = R l + t - p in r[0..3), r[3..6) = 0
KB_HD double prior_residual(int kind, const double *meas, const double *Om, const SE3 &T, double r[6]) {
    if (kind == PG_POSE_PRIOR) {
        const SE3 Zi{{meas[0], meas[1], meas[2], meas[3]}, {meas[4], meas[5], meas[6]}};
        se3_log(se3_mul(Zi, T), r);
    } else {
        const V3 a = se3_act(T, V3{meas[3], meas[4], meas[5]});
        r[0] = a.x - meas[0];
        r[1] = a.y - meas[1];
        r[2] = a.z - meas[2];
        r[3] = r[4] = r[5] = 0.0;
    }
    double s = 0.0;
    for (int a = 0; a < 6; ++a) {
        double o = 0.0;
        for (int b = 0; b < 6; ++b) o = o + Om[6 * a + b] * r[b];
        s = s + r[a] * o;
    }
    return s;
}

// dr/d delta of the right perturbation T Exp(delta), 6x6 row-major: J_r^-1(r) for a pose prior (the edge formula with
// T_i = I); [R, -R [l]x] in rows 0..2 and zeros below for a position prior (exact at delta = 0 for se3_exp)
KB_HD void prior_jacobian(int kind, const double *meas, const SE3 &T, const double r[6], double J[36]) {
    if (kind == PG_POSE_PRIOR) {
        se3_right_jacobian_inverse(r, J);
        return;
    }
    const M3 R = q_to_matrix(T.q);
    const double l[3] = {meas[3], meas[4], meas[5]};
    const double L[3][3] = {{0.0, -l[2], l[1]}, {l[2], 0.0, -l[0]}, {-l[1], l[0], 0.0}};
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 3; ++b) {
            J[6 * a + b] = R.m[a][b];
            J[6 * a + 3 + b] = -((R.m[a][0] * L[0][b] + R.m[a][1] * L[1][b]) + R.m[a][2] * L[2][b]);
        }
    for (int a = 18; a < 36; ++a) J[a] = 0.0;
}
