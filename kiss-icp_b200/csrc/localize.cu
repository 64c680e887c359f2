// The localizer's registration kernel, k_register_frame<LocalizeParams> (frame.cuh), in a translation unit of its own.
// A second kernel that calls the same __noinline__ ops inside api.cu's device module changes the code the compiler
// generates for the odometry kernel there; in a device module of its own it changes nothing.
// The headers are compiled here in a namespace of their own: the host side of a __device__ function or variable is an
// ordinary external symbol, and api.cu defines the same ones in kb. So this module also has its own copies of the
// device watchdog's words (device_ops.cuh), which host.cu arms with the others through localize_watchdog.
#define kb kb_localize
#include "frame.cuh"
#undef kb

namespace kb_localize {
template __global__ void k_register_frame<LocalizeParams>(const LocalizeParams P);
}

const void *localize_kernel() {
    return reinterpret_cast<const void *>(&kb_localize::k_register_frame<kb_localize::LocalizeParams>);
}

cudaError_t localize_watchdog(unsigned *d_host_words, const unsigned *init) { return kb_localize::watchdog_arm(d_host_words, init); }
