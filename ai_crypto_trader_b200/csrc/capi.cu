// C-ABI plumbing: error string, device check, launch counter.
#include <stdarg.h>
#include <string.h>
#include "common.cuh"

// Every struct of the C-ABI at the size its declaration in b200bt.h states (tests/test_abi_header.py holds the Python
// mirrors to the same layouts), so that a change to a struct that leaves its size comment behind fails the build.
static_assert(sizeof(b200bt_individual) == 40, "b200bt_individual layout");
static_assert(sizeof(b200bt_lane_stats) == 160, "b200bt_lane_stats layout");
static_assert(sizeof(b200bt_sweep_config) == 40, "b200bt_sweep_config layout");
static_assert(sizeof(b200bt_chunk_item) == 16, "b200bt_chunk_item layout");
static_assert(sizeof(b200bt_bt_params) == 56, "b200bt_bt_params layout");
static_assert(sizeof(b200bt_regime_params) == 64, "b200bt_regime_params layout");
static_assert(sizeof(b200bt_regime_window) == 64, "b200bt_regime_window layout");
static_assert(sizeof(b200bt_grid_individual) == 40, "b200bt_grid_individual layout");
static_assert(sizeof(b200bt_grid_regime_rule) == 24, "b200bt_grid_regime_rule layout");
static_assert(sizeof(b200bt_grid_stats) == 160, "b200bt_grid_stats layout");
static_assert(sizeof(b200bt_grid_service_stats) == 96, "b200bt_grid_service_stats layout");
static_assert(sizeof(b200bt_dca_individual) == 272, "b200bt_dca_individual layout");
static_assert(sizeof(b200bt_dca_stats) == 160, "b200bt_dca_stats layout");
static_assert(sizeof(b200bt_dca_service) == 40, "b200bt_dca_service layout");
static_assert(sizeof(b200bt_rl_agent) == 64, "b200bt_rl_agent layout");
static_assert(sizeof(b200bt_rl_agent_state) == 64, "b200bt_rl_agent_state layout");
static_assert(sizeof(b200bt_vp_params) == 32, "b200bt_vp_params layout");
static_assert(sizeof(b200bt_vp_row) == 384, "b200bt_vp_row layout");
static_assert(sizeof(b200bt_monitor_params) == 24, "b200bt_monitor_params layout");
static_assert(sizeof(b200bt_monitor_row) == 352, "b200bt_monitor_row layout");

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
