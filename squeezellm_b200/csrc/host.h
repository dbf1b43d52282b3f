// host.h - the host code every translation unit of the library shares: the error message of the last failed call, the process-wide
// state and its lock, the device set-up and launch of a kernel, the descriptor checks and the mode switches.  Every process-wide
// variable is defined once, in host.cu: a copy per unit would split the state (an error message or a mode switch would not reach
// the other units).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <initializer_list>
#include <mutex>
#include <vector>

#include "sqllm_b200.h"

// Every block of namespace sqllm is hidden: the units link to each other's host code, but the library does not export it.
namespace __attribute__((visibility("hidden"))) sqllm {

// records the message of a failed call for sqllm_last_error and returns `code`
int fail(int code, const char *fmt, ...);

// Process-wide state (mode switches, lazily read environment knobs, per-device state) is guarded by g_state_mu: the entry
// points may be called from several host threads.  Switching a mode (sqllm_set_deterministic / sqllm_set_lut_mode) while other
// threads are launching is allowed but takes effect per call; do not switch while a CUDA graph that should keep the old mode is
// being captured.
extern std::recursive_mutex g_state_mu;

struct DevInfo {
    int sm = 0;
    unsigned smem_raw = 0;               // shared-window address of dynamic shared memory; 0 until smem_window probes it
    std::vector<const void *> smem_set;  // kernels whose dynamic shared-memory limit dev_setup has raised
};
extern DevInfo g_dev[64];

// d.smem_raw, probed once per device (lutgemv.cu: the unit of the kernels that check the window)
int smem_window(DevInfo &d);

// A kernel and the dynamic shared memory it is launched with.
struct KernelSmem {
    const void *fn = nullptr;
    int bytes = 0;
    KernelSmem() = default;
    template <typename... P>
    KernelSmem(void (*f)(P...), int b) : fn((const void *)f), bytes(b) {}
};

// The device set-up of every launch, under g_state_mu: resolves the current device (its SM count is read once), raises the dynamic
// shared-memory limit of each kernel in `ks` (once per device), and returns the SM count in *sm and the shared-memory window in
// *smem_raw where asked (the window is probed on the first request, see smem_window).  `ks` is a braced list of KernelSmem, or an array.
template <typename List = std::initializer_list<KernelSmem>>
int dev_setup(const List &ks, int *sm = nullptr, unsigned *smem_raw = nullptr) {
    std::lock_guard<std::recursive_mutex> lk(g_state_mu);
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return fail(SQLLM_ECUDA, "cudaGetDevice failed");
    if (dev < 0 || dev >= 64) return fail(SQLLM_EINVAL, "device ordinal %d out of range", dev);
    DevInfo &d = g_dev[dev];
    if (d.sm == 0 && (cudaDeviceGetAttribute(&d.sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || d.sm <= 0)) {
        d.sm = 0;
        return fail(SQLLM_ECUDA, "cannot query SM count");
    }
    for (const KernelSmem &k : ks) {
        if (std::find(d.smem_set.begin(), d.smem_set.end(), k.fn) != d.smem_set.end()) continue;
        if (cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, k.bytes) != cudaSuccess)
            return fail(SQLLM_ECUDA, "cudaFuncSetAttribute failed: %s", cudaGetErrorString(cudaGetLastError()));
        d.smem_set.push_back(k.fn);
    }
    if (smem_raw) {
        const int rc = smem_window(d);
        if (rc) return rc;
        *smem_raw = d.smem_raw;
    }
    if (sm) *sm = d.sm;
    return SQLLM_OK;
}

// The one attribute of a cudaLaunchKernelEx launch: programmatic stream serialisation for the GEMV kernels that wait on the grid
// dependency (their prologue and weight stream overlap the previous kernel), cooperative for the sequence kernel (every CTA waits on
// every other one: they must all be resident), or a cluster of `cluster` CTAs along x for the kernels whose CTAs reduce through each
// other's shared memory.
struct LaunchAttr {
    int cluster;
    bool cooperative;
};
constexpr LaunchAttr PDL{0, false}, COOPERATIVE{0, true};
constexpr LaunchAttr cluster_of(int n) { return {n, false}; }

template <typename... P, typename... A>
cudaError_t launch_ex(void (*fn)(P...), dim3 grid, int block, int smem, cudaStream_t st, LaunchAttr la, const A &...args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr;
    if (la.cluster > 0) {
        attr.id = cudaLaunchAttributeClusterDimension;
        attr.val.clusterDim.x = la.cluster; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    } else if (la.cooperative) {
        attr.id = cudaLaunchAttributeCooperative;
        attr.val.cooperative = 1;
    } else {
        attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr.val.programmaticStreamSerializationAllowed = 1;
    }
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, fn, args...);
}

// The layer's buffers in a kernel's parameter struct (every one names them qw, lut, rows, cols, vals, full_rows, fri, topX): the
// dense rows only when both full_rows and topX > 0 are given, so that p.topX > 0 means "the layer has dense rows".
template <typename P>
void set_layer(P &p, const sqllm_lutgemv_args &a) {
    const bool hyb = a.full_rows && a.topX > 0;
    p.qw = reinterpret_cast<const uint32_t *>(a.qweight);
    p.lut = a.lookup_table;
    p.rows = a.rows; p.cols = a.cols; p.vals = a.vals;
    p.full_rows = hyb ? a.full_rows : nullptr;
    p.fri = hyb ? a.full_row_indices : nullptr;
    p.topX = hyb ? a.topX : 0;
}

// SQLLM_DT_F32, SQLLM_DT_F16 or SQLLM_DT_BF16
bool dt_valid(int dt);
int check_layer(const sqllm_lutgemv_args *a, int k_mult, int n_mult);
int check_common(const sqllm_lutgemv_args *a);

// the fused mode (1: deterministic, v1) and the table mode (1: fp16 pair table), from the environment until set through the C ABI
int det_mode();
int lut_mode();

// debug hooks (sqllm_debug_set_trace, sqllm_debug_last_grid): the next launch's timeline, and the grid of the last one-GEMV launch
extern int g_last_grid;
extern unsigned long long *g_trace;
extern size_t g_trace_stride;

// a 2-D tensor map over the packed matrix (rows x cols int32, boxes of 64 columns x box_rows), cached per (pointer, shape, box)
int get_tensor_map(const void *qweight, int rows, int cols, int box_rows, CUtensorMap &out);

// the *_batched symbols, and sqllm_lutgemv for batch >= 2 (lutgemv_rows.cu)
int launch_batched(const sqllm_lutgemv_args *a, cudaStream_t st);

}  // namespace sqllm
