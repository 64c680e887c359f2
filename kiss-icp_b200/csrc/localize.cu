// The localizer's registration kernel, k_register_frame<LocalizeParams> (frame.cuh), in a translation unit of its own.
// A second kernel that calls the same __noinline__ ops inside api.cu's device module changes the code the compiler
// generates for the odometry kernel there; in a device module of its own it changes nothing.
// The headers are compiled here in a namespace of their own: the host side of a __device__ function or variable is an
// ordinary external symbol, and api.cu defines the same ones in kb. So this module also has its own copies of the
// device watchdog's words (device_ops.cuh); api.cu sets and re-arms them, together with its own, through the functions
// below.
#define kb kb_localize
#include "frame.cuh"
#undef kb

namespace kb_localize {
template __global__ void k_register_frame<LocalizeParams>(const LocalizeParams P);
}

const void *localize_kernel() {
    return reinterpret_cast<const void *>(&kb_localize::k_register_frame<kb_localize::LocalizeParams>);
}

cudaError_t localize_watchdog_init(unsigned *d_host_words, const unsigned init[8]) {
    cudaError_t e = cudaMemcpyToSymbol(kb_localize::g_kb_wd_host, &d_host_words, sizeof(d_host_words));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(kb_localize::g_kb_wd, init, 8 * sizeof(unsigned));
    return e;
}

cudaError_t localize_watchdog_rearm() {
    const unsigned zero = 0;
    return cudaMemcpyToSymbol(kb_localize::g_kb_wd, &zero, sizeof(zero));
}
