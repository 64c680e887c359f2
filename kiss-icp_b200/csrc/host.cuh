// The host runtime every part of the C-ABI shares: error reporting, the calling thread's device, stream and grid
// settings, the device watchdog's host side, owners of CUDA resources and the execution context (Exec) that launches
// and waits. host.cu defines what is not a template or a small inline member; it contains no device code.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/kiss_icp_b200.h"
#include "types.cuh"

namespace kb_host {

using namespace kb_types;

#pragma GCC visibility push(hidden)  // (the library exports its C-ABI, not these)
extern thread_local std::string tl_err;  // kb_last_error
extern thread_local int tl_device;
extern thread_local cudaStream_t tl_user_stream;
extern thread_local int tl_grid_blocks;

// sets the calling thread's kb_last_error text; returns status
int fail(int status, const char *fmt, ...);

#define CK(call)                                                                              \
    do {                                                                                      \
        cudaError_t e_ = (call);                                                              \
        if (e_ != cudaSuccess) return fail(KB_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(e_)); \
    } while (0)
#define RET(call)              \
    do {                       \
        int s_ = (call);       \
        if (s_ != KB_OK) return s_; \
    } while (0)

int require_device();

// after a synchronisation: did a spin loop of the last launches give up (device_ops.cuh: the device watchdog)?
int watchdog_check(int device);
// a launch on this device never ended: every resource of the device is leaked from now on
void device_stuck(int device);
// a launch on this device (-1: any device) never ended
bool device_is_stuck(int device);
// where every CTA of the last k_register_frame was, read without waiting on the (stuck) compute stream
std::string phase_marks(int device);
#pragma GCC visibility pop

// Owner of one CUDA resource: device or pinned memory, an event, a stream. It records the device the resource was
// created on and releases it when it goes, unless a launch on that device never ended: cudaFree & co. would block
// forever then, so the resource is leaked with the stuck context. (The release calls find the resource's device from
// the handle: they do not depend on the current device.)
template <class H, cudaError_t (*Release)(H)>
struct Owned {
    H p = nullptr;
    int device = -1;  // where p was created
    Owned() = default;
    Owned(Owned &&o) noexcept { *this = std::move(o); }
    Owned &operator=(Owned &&o) noexcept {  // (o releases what this owned)
        std::swap(p, o.p);
        std::swap(device, o.device);
        return *this;
    }
    ~Owned() {
        if (p && !device_is_stuck(device)) Release(p);
    }

  protected:
    // release what this owns, then own what create(&handle) makes on the current device (nothing when it fails)
    template <class Create>
    cudaError_t make(Create create) {
        *this = Owned{};
        const cudaError_t e = create(&p);
        if (e == cudaSuccess)
            cudaGetDevice(&device);
        else
            p = nullptr;
        return e;
    }
};
struct Event : Owned<cudaEvent_t, cudaEventDestroy> {
    cudaError_t create(unsigned flags) { return make([&](cudaEvent_t *e) { return cudaEventCreateWithFlags(e, flags); }); }
};
struct Stream : Owned<cudaStream_t, cudaStreamDestroy> {
    cudaError_t create() { return make([](cudaStream_t *s) { return cudaStreamCreateWithFlags(s, cudaStreamNonBlocking); }); }
};
// the events ev[] on `device` (the current one): made anew unless the last, made last, is there already
template <size_t N>
int events_on(Event (&ev)[N], int device) {
    if (ev[N - 1].device != device)
        for (Event &e : ev) CK(e.create(cudaEventDefault));
    return KB_OK;
}

template <class T>
cudaError_t free_device(T *p) { return cudaFree(p); }
template <class T>
cudaError_t free_pinned(T *p) { return cudaFreeHost(p); }

// an array of n T in device memory, or in pinned host memory (Pinned)
template <class T, bool Pinned>
struct Buffer : Owned<T *, Pinned ? &free_pinned<T> : &free_device<T>> {
    size_t n = 0;
    Buffer() = default;
    Buffer(Buffer &&o) noexcept { *this = std::move(o); }
    Buffer &operator=(Buffer &&o) noexcept {
        Buffer::Owned::operator=(std::move(o));
        std::swap(n, o.n);
        return *this;
    }
    // exactly `count` elements; what the buffer held is released first
    cudaError_t alloc(size_t count) {
        const cudaError_t e = this->make([&](T **q) {
            return Pinned ? cudaHostAlloc(q, count * sizeof(T), cudaHostAllocDefault) : cudaMalloc(q, count * sizeof(T));
        });
        n = e == cudaSuccess ? count : 0;
        return e;
    }
    // at least `count` elements. Grown with 25% headroom: scan sizes jitter from frame to frame and a
    // cudaFree/cudaMalloc pair per new maximum would put milliseconds of allocator time on the hot path
    int ensure(size_t count) {
        if (count <= n) return KB_OK;
        const size_t want = std::max<size_t>(count + count / 4, 1024);
        const cudaError_t e = alloc(want);
        if (e != cudaSuccess)
            return fail(KB_ERR_CUDA, "%s of %zu bytes failed: %s", Pinned ? "cudaHostAlloc" : "cudaMalloc", want * sizeof(T),
                        cudaGetErrorString(e));
        return KB_OK;
    }
};
template <class T>
using DBuf = Buffer<T, false>;
template <class T>
using PinBuf = Buffer<T, true>;

// KB_TRACE_STALLS=<ms>: report host-side API calls of the frame paths that block longer than <ms> (diagnostic)
struct StallTrace {
    const char *what;
    std::chrono::steady_clock::time_point t0;
    static double limit_ms() {
        static const double v = [] {
            const char *e = std::getenv("KB_TRACE_STALLS");
            return e ? std::atof(e) : 0.0;
        }();
        return v;
    }
    explicit StallTrace(const char *w) : what(w) {
        if (limit_ms() > 0.0) t0 = std::chrono::steady_clock::now();
    }
    ~StallTrace() {
        if (limit_ms() > 0.0) {
            const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
            if (ms > limit_ms()) std::fprintf(stderr, "[kb stall] %s took %.1f ms\n", what, ms);
        }
    }
};

inline size_t pow2_at_least(size_t v) {
    size_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

// execution context: device, stream, persistent-grid size and the cross-CTA scratch
struct Exec {
    int device = 0;
    cudaStream_t stream = nullptr;
    Stream own_stream;  // (none when the calling thread set a stream: kb_set_stream)
    int grid = 0;
    int sms = 0;  // multiprocessors of the device
    Scratch sc{};  // all pointers null, profiling off
    TeamScratch team{};  // ll / out (qrec belongs to the caller's workspace)
    size_t icp_smem = 96 * 1024;  // dynamic shared memory of the ICP kernels: candidate coordinates of the team's source points (KB_ICP_SMEM_KB)
    int icp_team_q = TQ_PER_CTA;  // source points per CTA of the ICP team (KB_ICP_TEAM_Q; 0 = whole-grid ICP loop)
    unsigned tag_seq = 0;  // launch sequence number of the tagged ICP protocol
    unsigned long long launches = 0;
    bool bar_dirty = true;  // the barrier words may be non-zero (a kernel without Grid::finish() ran last)
    std::vector<const void *> smem_opted;  // kernels opted in to > 48 KB of dynamic shared memory on THIS context's device
    unsigned next_tag_base() { return (++tag_seq) << 13; }  // 8192 epochs per launch
    // a launch that uses more epochs (k_icp_batch) takes as many consecutive 8192-epoch blocks as it needs
    unsigned reserve_tags(size_t epochs) {
        const unsigned first = tag_seq + 1;
        tag_seq += static_cast<unsigned>((epochs + 8191) / 8192);
        return first << 13;
    }
    DBuf<uint4> batch_ll;  // all-gather regions of k_icp_batch's slots (allocated by the first batch call)
    std::vector<DBuf<char>> scratch_mem;  // what sc and team point to

    // `view` = a scratch array of `count` elements that lives as long as this context, zeroed on its stream when `zero`
    template <class T>
    int scratch(T *&view, size_t count, bool zero) {
        DBuf<char> b;
        CK(b.alloc(count * sizeof(T)));
        if (zero) CK(cudaMemsetAsync(b.p, 0, count * sizeof(T), stream));
        view = reinterpret_cast<T *>(b.p);
        scratch_mem.push_back(std::move(b));
        return KB_OK;
    }
    // on `dev`, on `user_stream` (nullptr: a stream of its own)
    int init(int dev, cudaStream_t user_stream);
    // opt in to > 48 KB of dynamic shared memory, once per kernel AND device (the attribute is per device)
    int opt_in_smem(const void *k, size_t bytes) {
        if (bytes <= 48 * 1024 || std::find(smem_opted.begin(), smem_opted.end(), k) != smem_opted.end()) return KB_OK;
        CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes)));
        smem_opted.push_back(k);
        return KB_OK;
    }
    template <class P>
    int coop(void (*kern)(P), const P &p, size_t smem = 0, bool self_reset = false) {
        return coop_raw(reinterpret_cast<const void *>(kern), const_cast<P *>(&p), smem, self_reset);
    }
    // `kern` takes one parameter struct, `param` points to it (a kernel of another device module: report_kernel())
    int coop_raw(const void *kern, void *param, size_t smem, bool self_reset) {
        CK(cudaSetDevice(device));
        RET(opt_in_smem(kern, smem));
        if (!self_reset || bar_dirty)  // kernels that end with Grid::finish() leave the barrier words zeroed themselves
            CK(cudaMemsetAsync(sc.bar, 0, BAR_WORDS * sizeof(unsigned), stream));
        bar_dirty = !self_reset;
        void *args[] = {param};
        CK(cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(BLOCK), args, smem, stream));
        ++launches;
        return KB_OK;
    }
    template <class A, class B>
    int coop(void (*kern)(A, B), const A &a, const B &b) {
        CK(cudaSetDevice(device));
        CK(cudaMemsetAsync(sc.bar, 0, BAR_WORDS * sizeof(unsigned), stream));
        bar_dirty = true;
        void *args[] = {const_cast<A *>(&a), const_cast<B *>(&b)};
        CK(cudaLaunchCooperativeKernel(reinterpret_cast<const void *>(kern), dim3(grid), dim3(BLOCK), args, 0, stream));
        ++launches;
        return KB_OK;
    }
    // wait for the stream with a deadline (KB_SYNC_TIMEOUT_S, default 30 s; 0 = wait forever): a launch that never
    // ends is reported as KB_ERR_CUDA instead of hanging the caller (the device watchdog should have fired long before)
    int sync();
    template <class Q>
    int wait_deadline(Q query, const char *what) {
        static const double limit_s = [] {
            const char *e = std::getenv("KB_SYNC_TIMEOUT_S");
            return e ? std::atof(e) : 30.0;
        }();
        const auto t0 = std::chrono::steady_clock::now();
        for (unsigned spins = 0;; ++spins) {
            const cudaError_t e = query();
            if (e == cudaSuccess) return KB_OK;
            if (e != cudaErrorNotReady) return fail(KB_ERR_CUDA, "%s wait failed: %s", what, cudaGetErrorString(e));
            if ((spins & 0x3ff) == 0x3ff && limit_s > 0.0 &&
                std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > limit_s) {
                const int wd = watchdog_check(device);
                device_stuck(device);
                if (wd != KB_OK) return wd;
                return fail(KB_ERR_CUDA, "the device did not finish the %s within %.0f s (launch %llu): giving up; %s", what, limit_s, launches,
                            phase_marks(device).c_str());
            }
        }
    }
};

// on the calling thread's device and stream (kb_set_device / kb_set_stream) unless given others
__attribute__((visibility("hidden"))) int make_exec(std::shared_ptr<Exec> *out, int device = tl_device,
                                                    cudaStream_t user_stream = tl_user_stream);

}  // namespace kb_host
