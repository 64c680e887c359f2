// The shared host runtime of the C-ABI (host.cuh) and the calls that configure it. No device code.
#include "host.cuh"

#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <mutex>

#pragma GCC visibility push(hidden)
// every device module that includes device_ops.cuh, by the function that sets its own copies of the watchdog's words
// (device_ops.cuh: watchdog_arm), named after its file; and where api.cu's module keeps its phase marks (g_kb_marks)
using WatchdogArm = cudaError_t(unsigned *d_host_words, const unsigned *init);
WatchdogArm core_watchdog, report_watchdog, relocalize_watchdog, probe_watchdog, pose_graph_watchdog, pose_graph_cov_watchdog,
    pose_graph_direct_watchdog, free_space_watchdog, degeneracy_watchdog, calib_watchdog, plane_adjust_watchdog;
const void *phase_marks_symbol();
#pragma GCC visibility pop

namespace kb_host {

thread_local std::string tl_err;
thread_local int tl_device = 0;
thread_local cudaStream_t tl_user_stream = nullptr;
thread_local int tl_grid_blocks = 0;

int fail(int status, const char *fmt, ...) {
    char buf[4096];  // (room for the per-CTA phase marks of the hang reports)
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    tl_err = buf;
    return status;
}


namespace {
int device_count() {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

WatchdogArm *const kWatchdogs[] = {core_watchdog,           report_watchdog,            relocalize_watchdog, probe_watchdog,
                                   pose_graph_watchdog,     pose_graph_cov_watchdog,    pose_graph_direct_watchdog,
                                   free_space_watchdog,     degeneracy_watchdog,        calib_watchdog,
                                   plane_adjust_watchdog};

// the device watchdog's report (device_ops.cuh): mapped host words per device, checked after every synchronisation
struct WatchdogHost {
    unsigned *host = nullptr;  // [0] flag [1] code [2] block [3] thread [4] a [5] b
};
WatchdogHost g_wd[64];
bool g_stuck[64];

// where every CTA of the last k_register_frame was (g_kb_marks)
std::string format_marks(const unsigned m[256]) {
    std::string out = "phase marks per CTA:";
    char buf[16];
    for (int i = 0; i < 160; ++i) {
        std::snprintf(buf, sizeof(buf), " %x", m[i]);
        out += buf;
    }
    return out;
}

int watchdog_init(int device) {
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    if (device < 0 || device >= 64 || g_wd[device].host) return KB_OK;
    unsigned *h = nullptr, *d = nullptr;
    CK(cudaHostAlloc(&h, 8 * sizeof(unsigned), cudaHostAllocMapped));
    std::memset(h, 0, 8 * sizeof(unsigned));
    CK(cudaHostGetDevicePointer(&d, h, 0));
    // give up after 2^24 polls (of the order of 10 s, below the host's 30 s deadline). 2^22 (a second or two) fired once in
    // ~40 full-file test runs at the FIRST grid barrier of a launch; whether that was a stall or a deadlock is not known.
    unsigned init[8] = {0, 0, 0, 0, 0, 0, 0, 24};
    if (const char *e = std::getenv("KB_WATCHDOG_SHIFT")) init[7] = static_cast<unsigned>(std::max(10, std::min(std::atoi(e), 31)));
    for (auto arm : kWatchdogs) CK(arm(d, init));
    g_wd[device].host = h;
    return KB_OK;
}
}  // namespace

int require_device() {
    return device_count() > 0 ? KB_OK : fail(KB_ERR_NO_DEVICE, "no CUDA device visible (this library has no CPU fallback)");
}
int watchdog_check(int device) {
    unsigned *h = (device >= 0 && device < 64) ? g_wd[device].host : nullptr;
    if (!h || !*reinterpret_cast<volatile unsigned *>(h)) return KB_OK;
    const unsigned code = h[1], block = h[2], thread = h[3], a = h[4], b = h[5];
    h[0] = 0;
    for (auto arm : kWatchdogs) arm(nullptr, nullptr);  // re-arm
    static const char *names[] = {"?", "grid barrier", "ICP gather", "ICP result record", "ICP team gather", "NN bulk copy"};
    std::string marks;
    unsigned m[256];
    if (cudaMemcpyFromSymbol(m, phase_marks_symbol(), sizeof(m), 0, cudaMemcpyDeviceToHost) == cudaSuccess)
        marks = "; " + format_marks(m);  // (the launch has ended: a plain copy)
    cudaGetLastError();
    return fail(KB_ERR_CUDA, "device watchdog: a kernel gave up waiting at the %s (block %u, thread %u, a=%u, b=%u; grid barrier: a = target, b = counter); "
                             "the results of that launch are invalid%s",
                names[code < 6 ? code : 0], block, thread, a, b, marks.c_str());
}

void device_stuck(int device) {
    if (device >= 0 && device < 64) g_stuck[device] = true;
}
bool device_is_stuck(int device) {
    if (device < 0) {
        for (bool b : g_stuck)
            if (b) return true;
        return false;
    }
    return device < 64 && g_stuck[device];
}
std::string phase_marks(int device) {
    // the compute stream is stuck: read the marks on a stream of their own (bounded wait, the copy engine is free)
    unsigned marks[256];
    cudaStream_t side = nullptr;
    if (cudaSetDevice(device) != cudaSuccess || cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking) != cudaSuccess) return "";
    std::string out;
    if (cudaMemcpyFromSymbolAsync(marks, phase_marks_symbol(), sizeof(marks), 0, cudaMemcpyDeviceToHost, side) == cudaSuccess) {
        const auto t0 = std::chrono::steady_clock::now();
        cudaError_t q;
        while ((q = cudaStreamQuery(side)) == cudaErrorNotReady &&
               std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() < 5.0) {
        }
        out = q == cudaSuccess ? format_marks(marks) : "(phase marks unreadable)";
    }
    return out;  // (the side stream is leaked with the rest of the stuck context)
}

int Exec::init(int dev, cudaStream_t user_stream) {
    RET(require_device());
    device = dev;
    CK(cudaSetDevice(device));
    RET(watchdog_init(device));
    if (user_stream) {
        stream = user_stream;
    } else {
        CK(own_stream.create());
        stream = own_stream.p;
    }
    int coop = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    CK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device));
    if (!coop) return fail(KB_ERR_CUDA, "device does not support cooperative launch");
    grid = tl_grid_blocks > 0 ? std::min(tl_grid_blocks, sms) : sms;
    grid = std::min(grid, 256);  // the two-level gather tree of the ICP loop handles up to 16 x 16 CTAs
    RET(scratch(sc.bar, BAR_WORDS, true));
    RET(scratch(sc.blk_d, 2 * grid * NPART, false));
    RET(scratch(sc.blk_i, 2 * grid, false));
    RET(scratch(sc.ll_part, NPART * grid, true));
    RET(scratch(sc.ll_res, LL_RES, true));
    RET(scratch(sc.ll_group, NPART * 16, true));
    RET(scratch(team.ll, 2 * NPART * TEAM_MAX * TEAM_MAX, true));  // 11 MB: one copy of the partials per reader
    RET(scratch(team.out, 16, false));
    RET(scratch(sc.dbg, 64 + 4 * grid, true));
    if (const char *e = std::getenv("KB_ICP_TEAM_Q")) icp_team_q = std::max(0, std::min(std::atoi(e), TQ_MAX));
    if (const char *e = std::getenv("KB_ICP_SMEM_KB")) icp_smem = static_cast<size_t>(std::max(60, std::min(std::atoi(e), 180))) * 1024;
    team.smem_bytes = static_cast<int>(icp_smem);
    team.radius_frac = 0.2;
    if (const char *e = std::getenv("KB_ICP_RADIUS")) team.radius_frac = std::max(0.01, std::min(std::atof(e), 0.45));
    return KB_OK;
}

int Exec::sync() {
    RET(wait_deadline([&] { return cudaStreamQuery(stream); }, "stream"));
    return watchdog_check(device);
}

int make_exec(std::shared_ptr<Exec> *out, int device, cudaStream_t user_stream) {
    auto e = std::make_shared<Exec>();
    RET(e->init(device, user_stream));
    *out = e;
    return KB_OK;
}

}  // namespace kb_host

using namespace kb_host;

extern "C" {

const char *kb_last_error(void) { return tl_err.c_str(); }
const char *kb_version(void) { return "kiss_icp_b200 0.1 (sm_90a)"; }
int kb_device_count(void) { return device_count(); }
int kb_set_device(int device) {
    if (device < 0 || device >= device_count()) return fail(KB_ERR_INVALID_ARG, "device %d out of range", device);
    tl_device = device;
    return KB_OK;
}
int kb_set_stream(void *cuda_stream) {
    tl_user_stream = static_cast<cudaStream_t>(cuda_stream);
    return KB_OK;
}
int kb_set_grid_blocks(int blocks) {
    if (blocks < 0) return fail(KB_ERR_INVALID_ARG, "blocks < 0");
    tl_grid_blocks = blocks;
    return KB_OK;
}
int kb_any_device_stuck(void) { return device_is_stuck(-1) ? 1 : 0; }

}  // extern "C"
