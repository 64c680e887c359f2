// The kernels of degeneracy-aware ICP (frame.cuh: degen_form, DESIGN.md section 4.16), in a device module of their own
// for the reason report.cu gives: a kernel that calls the same __noinline__ ops inside another module changes the code
// generated for the kernels already there. Like report.cu, the headers are compiled in a namespace of their own, with
// this module's own copies of the device watchdog's words (armed by host.cu through degeneracy_watchdog).
//   k_register_frame<DegenParams, localizer, planes>  a localizer or an odometry pipeline with a degeneracy ratio (both
//                                                     report fits), with or without plane reporting
#define kb kb_degen
#include "frame.cuh"
#undef kb

namespace kb_degen {
template __global__ void k_register_frame<DegenParams, false, false>(const __grid_constant__ DegenParams P);
template __global__ void k_register_frame<DegenParams, false, true>(const __grid_constant__ DegenParams P);
template __global__ void k_register_frame<DegenParams, true, false>(const __grid_constant__ DegenParams P);
template __global__ void k_register_frame<DegenParams, true, true>(const __grid_constant__ DegenParams P);
}  // namespace kb_degen

const void *degeneracy_kernel(bool localizer, bool planes) {
    using kb_degen::DegenParams;
    using kb_degen::k_register_frame;
    static const void *const kernels[2][2] = {
        {reinterpret_cast<const void *>(&k_register_frame<DegenParams, false, false>),
         reinterpret_cast<const void *>(&k_register_frame<DegenParams, false, true>)},
        {reinterpret_cast<const void *>(&k_register_frame<DegenParams, true, false>),
         reinterpret_cast<const void *>(&k_register_frame<DegenParams, true, true>)}};
    return kernels[localizer][planes];
}

cudaError_t degeneracy_watchdog(unsigned *d_host_words, const unsigned *init) {
    return kb_degen::watchdog_arm(d_host_words, init);
}
