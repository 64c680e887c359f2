// The kernels that report plane constraints (frame.cuh: op_fit_planes), in a translation unit of their own, for the
// reason localize.cu gives: inside another device module further instantiations would change the code the compiler
// generates for the kernels every other pipeline runs. Like localize.cu, it compiles the headers in a namespace of its
// own and has its own copies of the device watchdog's words, which host.cu arms through constraints_watchdog.
//   k_register_frame<LocalizeConstraintParams>  a localizer with plane reporting on
//   k_register_frame<OdometryConstraintParams>  an odometry pipeline with fit and plane reporting on
//   k_constraints                               kb_registration_constraints: the same pass for one source at one pose
#define kb kb_constraints
#include "frame.cuh"
#undef kb

namespace kb_constraints {
template __global__ void k_register_frame<LocalizeConstraintParams>(const LocalizeConstraintParams P);
template __global__ void k_register_frame<OdometryConstraintParams>(const OdometryConstraintParams P);

// cooperative: the pass, one grid barrier, the partials added by the last CTA (as in the pipeline kernels)
__global__ void __launch_bounds__(BLOCK, 1) k_constraints(const ConstraintsParams P) {
    __shared__ Shared sh;
    Grid g;
    g.init(P.sc.bar);
    op_fit_planes<false>(sh, P.m, P.src, P.n, P.pose, P.max_dist, 0.0, nullptr, P.planes.part);
    g.sync();
    if (blockIdx.x == gridDim.x - 1) planes_finish(P.planes);
    g.finish();
}
}  // namespace kb_constraints

const void *localize_constraints_kernel() {
    return reinterpret_cast<const void *>(&kb_constraints::k_register_frame<kb_constraints::LocalizeConstraintParams>);
}
const void *odometry_constraints_kernel() {
    return reinterpret_cast<const void *>(&kb_constraints::k_register_frame<kb_constraints::OdometryConstraintParams>);
}
const void *constraints_kernel() { return reinterpret_cast<const void *>(&kb_constraints::k_constraints); }

cudaError_t constraints_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_constraints::watchdog_arm(d_host_words, init); }
