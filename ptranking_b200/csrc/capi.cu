// capi.cu -- bookkeeping entry points of the C ABI (error string, launch counter, device check).
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "common.cuh"

namespace ptrb200 {

static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return PTRB200_ERR_CUDA;
    }
    return PTRB200_OK;
}

// ---- per-launch event timing ------------------------------------------------
struct TimedLaunch { const char* tag; cudaEvent_t a, b; };
static bool g_timing = false;
static std::vector<TimedLaunch> g_timed;

bool timing_enabled() { return g_timing; }
void timing_before(const char* tag, cudaStream_t st) {
    TimedLaunch t;
    t.tag = tag;
    cudaEventCreate(&t.a);
    cudaEventCreate(&t.b);
    cudaEventRecord(t.a, st);
    g_timed.push_back(t);
}
void timing_after(cudaStream_t st) { cudaEventRecord(g_timed.back().b, st); }

}  // namespace ptrb200

extern "C" {

int ptrb200_timing_enable(int on) {
    ptrb200::g_timing = on != 0;
    return PTRB200_OK;
}

int ptrb200_timing_report(char* buf, int buflen) {
    using namespace ptrb200;
    if (!buf || buflen <= 0) { set_error("timing_report: bad buffer"); return PTRB200_ERR_INVALID; }
    std::map<std::string, std::pair<int, double>> acc;
    for (auto& t : g_timed) {
        cudaEventSynchronize(t.b);
        float ms = 0.0f;
        cudaEventElapsedTime(&ms, t.a, t.b);
        auto& e = acc[t.tag];
        e.first += 1;
        e.second += ms;
        cudaEventDestroy(t.a);
        cudaEventDestroy(t.b);
    }
    g_timed.clear();
    std::string out;
    char line[256];
    for (auto& kv : acc) {
        snprintf(line, sizeof(line), "%s\t%d\t%.6f\n", kv.first.c_str(), kv.second.first, kv.second.second);
        out += line;
    }
    if ((int)out.size() + 1 > buflen) { set_error("timing_report: buffer too small (%zu needed)", out.size() + 1); return PTRB200_ERR_WORKSPACE; }
    memcpy(buf, out.c_str(), out.size() + 1);
    return PTRB200_OK;
}

int ptrb200_version(void) { return 101; }

const char* ptrb200_last_error(void) { return ptrb200::g_err; }

unsigned long long ptrb200_launch_count(void) { return ptrb200::g_launches.load(std::memory_order_relaxed); }

int ptrb200_device_ok(void) {
    int dev = 0;
    cudaDeviceProp prop;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
        ptrb200::set_error("no CUDA device: %s", cudaGetErrorString(cudaGetLastError()));
        return 0;
    }
    if (prop.major != 9 || prop.minor != 0) {
        ptrb200::set_error("device %s is sm_%d%d; this library is built for sm_90a only", prop.name, prop.major, prop.minor);
        return 0;
    }
    return 1;
}

}  // extern "C"
