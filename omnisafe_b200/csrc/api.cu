// C-ABI plumbing shared by all entry points: error string, version, device query.
#include "common.cuh"
#include <mutex>
#include <string.h>

static thread_local char g_err[1024] = "";

extern "C" {

void osb_set_error(const char* msg) {
    strncpy(g_err, msg ? msg : "", sizeof(g_err) - 1);
    g_err[sizeof(g_err) - 1] = 0;
}

const char* osb_last_error(void) { return g_err; }

int osb_abi_version(void) { return 1; }

static long long g_launches = 0;
void osb_count_launch(void) { ++g_launches; }
// number of kernels this library has launched in this process (every launch site counts itself)
long long osb_launch_count(void) { return g_launches; }

// Fills sm_count / cc_major / cc_minor of `device`; fails loudly when there is no CUDA device.
int osb_device_info(int device, int* sm_count, int* cc_major, int* cc_minor) {
    cudaDeviceProp prop;
    OSB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    return OSB_OK;
}

}  // extern "C"

namespace osb {

// Device scratch for the tensor-core accumulator images (csrc/umma.cuh): one buffer per (device, slot), grown on
// demand.  A buffer that has been handed out is never freed (growth allocates a new one and keeps the old one for the
// life of the process), so a pointer stays valid for the launch it was fetched for and no growth synchronises the device.
// Contract: the launches of one kernel family on one device share its buffer, so they must be ordered on one stream;
// growth calls cudaMalloc, which CUDA-graph capture does not allow -- run a launch of the same size before capturing it
// (acc_scratch_capacity tells whether a launch would grow the buffer).
static constexpr int MAX_DEV = 64;
static std::mutex mu;
static float* buf[MAX_DEV][ACC_SLOTS] = {};
static size_t cap[MAX_DEV][ACC_SLOTS] = {};

float* acc_scratch(int slot, size_t bytes) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAX_DEV || slot < 0 || slot >= ACC_SLOTS) {
        osb_set_error("acc_scratch: bad device or slot");
        return nullptr;
    }
    std::lock_guard<std::mutex> lock(mu);
    if (cap[dev][slot] < bytes) {
        const size_t grown = bytes > 2 * cap[dev][slot] ? bytes : 2 * cap[dev][slot];   // geometric: few retired buffers
        void* ptr = nullptr;
        const cudaError_t e = cudaMalloc(&ptr, grown);
        if (e != cudaSuccess) {
            char msg[256];
            snprintf(msg, sizeof(msg), "acc_scratch: cudaMalloc(%zu) -> %s", grown, cudaGetErrorString(e));
            osb_set_error(msg);
            return nullptr;
        }
        buf[dev][slot] = static_cast<float*>(ptr);
        cap[dev][slot] = grown;
    }
    return buf[dev][slot];
}

size_t acc_scratch_capacity(int slot) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= MAX_DEV || slot < 0 || slot >= ACC_SLOTS) return 0;
    std::lock_guard<std::mutex> lock(mu);
    return cap[dev][slot];
}

int grid_sms() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
        return 1;
    return n < MAX_GRID_CTAS ? n : MAX_GRID_CTAS;
}

}  // namespace osb
