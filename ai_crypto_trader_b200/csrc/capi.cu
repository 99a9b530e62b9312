// C-ABI plumbing: error string, device check, launch counter.
#include <stdarg.h>
#include <string.h>
#include "common.cuh"

namespace b200bt {

static thread_local char t_err[512] = "";
std::atomic<int64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(t_err, sizeof(t_err), fmt, ap);
    va_end(ap);
}

// The library is compiled for sm_90a (H100) only; anything else cannot run its kernels.
int check_device() {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        set_error("no CUDA device: %s", cudaGetErrorString(e));
        cudaGetLastError();
        return B200BT_ENODEVICE;
    }
    static thread_local int ok_dev = -1;
    if (ok_dev == dev) return B200BT_OK;
    int major = 0;
    e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    if (e != cudaSuccess || major != 9) {
        set_error("device %d is not sm_90 (compute capability major %d); this library has no other code path", dev, major);
        cudaGetLastError();
        return B200BT_ENODEVICE;
    }
    ok_dev = dev;
    return B200BT_OK;
}

int device_sm_count() {
    int dev = 0, sms = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        sms <= 0) {
        cudaGetLastError();
        return 132;
    }
    return sms;
}

}  // namespace b200bt

extern "C" {

int b200bt_abi_version(void) { return B200BT_ABI_VERSION; }
const char* b200bt_last_error(void) { return b200bt::t_err; }
int64_t b200bt_launch_count(void) { return b200bt::g_launches.load(); }

}
