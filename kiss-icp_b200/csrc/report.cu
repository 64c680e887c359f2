// The kernels that report fits and plane constraints (frame.cuh: op_fit_planes), in a translation unit of their own.
// A further kernel that calls the same __noinline__ ops inside api.cu's device module changes the code the compiler
// generates for the odometry kernel there; in a device module of its own it changes nothing.
// The headers are compiled here in a namespace of their own: the host side of a __device__ function or variable is an
// ordinary external symbol, and api.cu defines the same ones in kb. So this module also has its own copies of the
// device watchdog's words (device_ops.cuh), which host.cu arms with the others through report_watchdog.
//   k_register_frame<ReportParams, localizer, planes>  a localizer, or an odometry pipeline with fit reporting on,
//                                                      with or without plane reporting
//   k_pose_pass<true, false>                           kb_registration_build_system: the fit of one source at one pose
//   k_pose_pass<false, true>                           kb_registration_constraints: the plane pass for one source at
//                                                      one pose
#define kb kb_report
#include "frame.cuh"
#undef kb

namespace kb_report {
template __global__ void k_register_frame<ReportParams, false, false>(const __grid_constant__ ReportParams P);
template __global__ void k_register_frame<ReportParams, false, true>(const __grid_constant__ ReportParams P);
template __global__ void k_register_frame<ReportParams, true, false>(const __grid_constant__ ReportParams P);
template __global__ void k_register_frame<ReportParams, true, true>(const __grid_constant__ ReportParams P);

// cooperative: the pass, one grid barrier, the partials added by the last CTA (as in the pipeline kernels)
template <bool FIT, bool PLANES>
__global__ void __launch_bounds__(BLOCK, 1) k_pose_pass(const PosePassParams P) {
    __shared__ Shared sh;
    Grid g;
    g.init(P.sc.bar);
    op_fit_planes<FIT, PLANES>(sh, P.m, P.src, P.n, P.pose, P.max_dist, P.kscale, P.fit.part, P.planes.part);
    g.sync();
    if (blockIdx.x == gridDim.x - 1) {
        if constexpr (FIT) fit_finish(P.fit, P.n);
        if constexpr (PLANES) planes_finish(P.planes);
    }
    g.finish();
}
template __global__ void k_pose_pass<true, false>(const PosePassParams P);
template __global__ void k_pose_pass<false, true>(const PosePassParams P);
}  // namespace kb_report

const void *report_kernel(bool localizer, bool planes) {
    using kb_report::k_register_frame;
    using kb_report::ReportParams;
    static const void *const kernels[2][2] = {
        {reinterpret_cast<const void *>(&k_register_frame<ReportParams, false, false>),
         reinterpret_cast<const void *>(&k_register_frame<ReportParams, false, true>)},
        {reinterpret_cast<const void *>(&k_register_frame<ReportParams, true, false>),
         reinterpret_cast<const void *>(&k_register_frame<ReportParams, true, true>)}};
    return kernels[localizer][planes];
}
const void *pose_pass_kernel(bool fit) {
    using kb_report::k_pose_pass;
    return fit ? reinterpret_cast<const void *>(&k_pose_pass<true, false>)
               : reinterpret_cast<const void *>(&k_pose_pass<false, true>);
}

cudaError_t report_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_report::watchdog_arm(d_host_words, init); }
