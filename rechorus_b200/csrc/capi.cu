// capi.cu -- version / error / measurement entry points of libb200rec.so
#include "common.cuh"

namespace b2r {

static thread_local char g_err[512] = "";

char* err_buf() { return g_err; }

int set_error(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

int sm_count() {
    static thread_local int cached_dev = -1;
    static thread_local int cached_sms = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev != cached_dev) {
        int sms = 0;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
        cached_dev = dev;
        cached_sms = sms;
    }
    return cached_sms;
}

static long long g_launches = 0;
static cudaEvent_t g_prof_start[B2R_PROF_TAGS] = {nullptr};
static cudaEvent_t g_prof_stop[B2R_PROF_TAGS] = {nullptr};

void count_launch() { __atomic_add_fetch(&g_launches, 1, __ATOMIC_RELAXED); }

void profile_begin(int tag, cudaStream_t s) {
    if (tag >= 0 && tag < B2R_PROF_TAGS && g_prof_start[tag]) cudaEventRecord(g_prof_start[tag], s);
}

void profile_end(int tag, cudaStream_t s) {
    if (tag >= 0 && tag < B2R_PROF_TAGS && g_prof_stop[tag]) {
        cudaEventRecord(g_prof_stop[tag], s);
        g_prof_start[tag] = nullptr;     // one-shot: re-arm before the next call
        g_prof_stop[tag] = nullptr;
    }
}

}  // namespace b2r

extern "C" long long b2r_launch_count(void) { return __atomic_load_n(&b2r::g_launches, __ATOMIC_RELAXED); }

extern "C" int b2r_profile_arm(int tag, void* ev_start, void* ev_stop) {
    B2R_REQUIRE(tag >= 0 && tag < B2R_PROF_TAGS, B2R_E_BADARG, "b2r_profile_arm: tag %d", tag);
    b2r::g_prof_start[tag] = reinterpret_cast<cudaEvent_t>(ev_start);
    b2r::g_prof_stop[tag] = reinterpret_cast<cudaEvent_t>(ev_stop);
    return 0;
}

extern "C" int b2r_version(void) { return B2R_VERSION; }

extern "C" const char* b2r_last_error(void) { return b2r::err_buf(); }
