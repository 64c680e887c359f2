// The registration kernel of an odometry pipeline that reports fits, k_register_frame<OdometryFitParams> (frame.cuh), in
// a translation unit of its own, for the reason localize.cu gives: inside api.cu's device module a further instantiation
// would change the code the compiler generates for the odometry kernel every other pipeline runs. Like localize.cu, it
// compiles the headers in a namespace of its own and has its own copies of the device watchdog's words, which api.cu
// sets and re-arms through the functions below.
#define kb kb_odometry_fit
#include "frame.cuh"
#undef kb

namespace kb_odometry_fit {
template __global__ void k_register_frame<OdometryFitParams>(const OdometryFitParams P);
}

const void *odometry_fit_kernel() {
    return reinterpret_cast<const void *>(&kb_odometry_fit::k_register_frame<kb_odometry_fit::OdometryFitParams>);
}

cudaError_t odometry_fit_watchdog_init(unsigned *d_host_words, const unsigned init[8]) {
    cudaError_t e = cudaMemcpyToSymbol(kb_odometry_fit::g_kb_wd_host, &d_host_words, sizeof(d_host_words));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(kb_odometry_fit::g_kb_wd, init, 8 * sizeof(unsigned));
    return e;
}

cudaError_t odometry_fit_watchdog_rearm() {
    const unsigned zero = 0;
    return cudaMemcpyToSymbol(kb_odometry_fit::g_kb_wd, &zero, sizeof(zero));
}
