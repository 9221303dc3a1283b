// Shared helpers for libcouncil_b200.so (sm_90a).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include "../../include/council_b200.h"

namespace cg {

void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;
// kernel-selection switches of cg_set_tensor_core_mode: per calling THREAD (like cg_last_error), not process-global
extern thread_local int g_tc_mode;
extern thread_local int g_small_bn;
extern thread_local int g_wgrad_tma;
extern thread_local int g_tc_serial_epilogue;
extern thread_local int g_tc_reg_epilogue;

constexpr int CG_MAX_DEVICES = 64;
inline int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return dev >= 0 && dev < CG_MAX_DEVICES ? dev : 0;
}
// true exactly once per (call site flag array, device): per-function attributes and occupancy queries are per device
struct PerDeviceOnce {
    std::atomic<bool> done[CG_MAX_DEVICES];
    bool first() { return !done[current_device()].exchange(true); }
    void reset() { done[current_device()].store(false); }
};

inline int check_launch(const char* what) {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return CG_ERR_CUDA;
    }
    return CG_OK;
}

#define CG_REQUIRE(cond, ...)                \
    do {                                     \
        if (!(cond)) {                       \
            cg::set_error(__VA_ARGS__);      \
            return CG_ERR_ARG;               \
        }                                    \
    } while (0)

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

// ---- programmatic dependent launch (PDL) --------------------------------------------------------------------------------------------
// A training step is ~670 short-to-medium kernels in one stream.  Every kernel of this library (a) lets its successor start launching
// at once (griddepcontrol.launch_dependents as its first instruction: CTAs of the next kernel are scheduled as SM resources free up and run
// their on-chip prologue -- barrier init, tensor-map prefetch) and (b) executes griddepcontrol.wait before it touches
// global memory: that blocks until the WHOLE preceding grid has completed and its writes are visible, so the data dependences are
// exactly those of plain stream order (every kernel waits, so completion is transitive along the stream).  Kernels of other libraries
// (NCCL, memsets, copies) are launched without the attribute and keep full stream serialisation on both sides.
// Early-scheduled dependents cost more than the launch gaps they hide once kernels are long, so the attribute is OFF unless mode
// bit 22 asks for it (the trainer does on small, launch-bound maps).
extern thread_local int g_pdl;
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline void launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = g_pdl;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    (void)cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);  // errors surface through check_launch()'s cudaGetLastError
}

__device__ __forceinline__ float apply_act(float v, int act, float slope) {
    if (act == CG_ACT_RELU) return v > 0.f ? v : 0.f;
    if (act == CG_ACT_LRELU) return v > 0.f ? v : v * slope;
    if (act == CG_ACT_TANH) return tanhf(v);
    return v;
}

// geometry helpers shared by host code
struct ConvDims {
    int Hin, Win;   // size the convolution sees (after optional x2 upsample)
    long Mpix;      // B*Ho*Wo
    int Ktot;       // KH*KW*Cin
};
inline ConvDims conv_dims(const cg_conv_geom& g) {
    ConvDims d;
    d.Hin = g.ups ? 2 * g.H : g.H;
    d.Win = g.ups ? 2 * g.W : g.W;
    d.Mpix = (long)g.B * g.Ho * g.Wo;
    d.Ktot = g.KH * g.KW * g.Cin;
    return d;
}
int validate_geom(const cg_conv_geom& g);

// ---- SIMT fp32 implicit-GEMM convolutions (conv_simt.cu) ----
int simt_conv_fwd(const cg_conv_geom& g, const float* x, const float* w, const float* bias, float* y,
                  int act, float slope, cudaStream_t st);
// writes gradient w.r.t. the tensor the convolution SEES (upsampled size if g.ups)
int simt_conv_dgrad(const cg_conv_geom& g, const float* dy, const float* w, float* dx_seen,
                    const float* addend, const float* mask_src, float mask_slope, cudaStream_t st);
int simt_conv_wgrad(const cg_conv_geom& g, const float* x, const float* dy, float* dw, void* ws,
                    size_t ws_bytes, cudaStream_t st);
size_t simt_wgrad_ws(const cg_conv_geom& g);
int colsum(const float* dy, float* db, int G, long rows, int C, void* ws, size_t ws_bytes, cudaStream_t st);
size_t colsum_ws(int G, long rows, int C);
int pool2x2_sum(const float* d_up, float* dx, const float* addend, const float* mask_src, float mask_slope,
                long N, int H, int W, int C, cudaStream_t st);

// ---- TF32 tensor-core implicit-GEMM convolutions (conv_tc.cu) ----
bool tc_fwd_supported(const cg_conv_geom& g);
int tc_conv_fwd(const cg_conv_geom& g, const float* x, const float* w, const float* bias, float* y,
                int act, float slope, void* ws, size_t ws_bytes, cudaStream_t st, float* stats_part = nullptr);
int tc_fwd_stats_chunks(const cg_conv_geom& g);
int in_stats_finalize(const float* part, float* mean, float* rstd, long GBC, int nchunks, int HW, float eps, cudaStream_t st);
size_t tc_fwd_ws(const cg_conv_geom& g);
bool tc_dgrad_supported(const cg_conv_geom& g);
size_t tc_dgrad_ws(const cg_conv_geom& g);
int tc_conv_dgrad(const cg_conv_geom& g, const float* dy, const float* w, float* dx, const float* addend,
                  const float* mask_src, float mask_slope, void* ws, size_t ws_bytes, cudaStream_t st);

bool tc_wgrad_supported(const cg_conv_geom& g);
size_t tc_wgrad_ws(const cg_conv_geom& g);
int tc_conv_wgrad(const cg_conv_geom& g, const float* x, const float* dy, float* dw, void* ws, size_t ws_bytes,
                  cudaStream_t st);

int tc_sm_count();
void tc_map_cache_stats(uint64_t* hits, uint64_t* misses);

// ---- vector-shaped layers (512 -> 1 patch heads, the MLP's wide output layer) as streaming fp32 kernels (conv_small.cu) ----
bool small_fwd_supported(const cg_conv_geom& g, int act);
bool small_dgrad_supported(const cg_conv_geom& g);
bool small_wgrad_supported(const cg_conv_geom& g);
size_t small_ws(const cg_conv_geom& g, int which);
int small_conv_fwd(const cg_conv_geom& g, const float* x, const float* w, const float* bias, float* y, cudaStream_t st);
int small_conv_dgrad(const cg_conv_geom& g, const float* dy, const float* w, float* dx, const float* addend, const float* mask_src,
                     float slope, void* ws, size_t ws_bytes, cudaStream_t st);
int small_conv_wgrad(const cg_conv_geom& g, const float* x, const float* dy, float* dw, float* db, void* ws, size_t ws_bytes, cudaStream_t st);

}  // namespace cg
