// The registration kernel of an odometry pipeline that reports fits, k_register_frame<OdometryFitParams> (frame.cuh), in
// a translation unit of its own, for the reason localize.cu gives: inside api.cu's device module a further instantiation
// would change the code the compiler generates for the odometry kernel every other pipeline runs. Like localize.cu, it
// compiles the headers in a namespace of its own and has its own copies of the device watchdog's words, which host.cu
// arms through odometry_fit_watchdog.
#define kb kb_odometry_fit
#include "frame.cuh"
#undef kb

namespace kb_odometry_fit {
template __global__ void k_register_frame<OdometryFitParams>(const OdometryFitParams P);
}

const void *odometry_fit_kernel() {
    return reinterpret_cast<const void *>(&kb_odometry_fit::k_register_frame<kb_odometry_fit::OdometryFitParams>);
}

cudaError_t odometry_fit_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_odometry_fit::watchdog_arm(d_host_words, init); }
