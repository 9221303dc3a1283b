// C-ABI entry points: error reporting, device info and the convolution dispatch.
#include "common.cuh"
#include <string.h>

namespace cg {

static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};
thread_local int g_tc_mode = 7;
thread_local int g_pdl = 0;  // programmatic dependent launch between this library's kernels (mode bit 22 sets it)

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int validate_geom(const cg_conv_geom& g) {
    CG_REQUIRE(g.G >= 1 && (g.x_groups == 1 || g.x_groups == g.G), "conv: x_groups=%d must be 1 or G=%d", g.x_groups, g.G);
    CG_REQUIRE(g.Cin % 4 == 0 && g.Cin > 0, "conv: Cin=%d must be a positive multiple of 4", g.Cin);
    CG_REQUIRE(g.Cout > 0 && g.B > 0 && g.H > 0 && g.W > 0, "conv: empty tensor");
    CG_REQUIRE(g.stride >= 1 && g.KH >= 1 && g.KW >= 1 && g.pad >= 0, "conv: bad kernel geometry");
    int Hin = g.ups ? 2 * g.H : g.H, Win = g.ups ? 2 * g.W : g.W;
    int Ho = (Hin + 2 * g.pad - g.KH) / g.stride + 1, Wo = (Win + 2 * g.pad - g.KW) / g.stride + 1;
    CG_REQUIRE(Ho == g.Ho && Wo == g.Wo, "conv: output size %dx%d inconsistent with geometry (expected %dx%d)", g.Ho, g.Wo, Ho, Wo);
    return CG_OK;
}

// ---- patch path for the image-side layers (Cin <= 8: 3/4-lane images, the 8-lane council-D pair) -----------
// TMA im2col moves 16..32 bytes per pixel-tap for these layers and is request-bound, so their (tiny) input is
// expanded once into an explicit patch matrix P[pixel][KH*KW*Cin padded to 32k] and the layer runs as a 1x1
// convolution on the tensor path.  P is 96..224 floats per pixel -- small next to the 64-channel output.
static bool patch_path(const cg_conv_geom& g) {
    if (!g_tc_mode || g.ups || g.Cin > 8 || g.Cout % 32 != 0) return false;
    int k2p = (g.KH * g.KW * g.Cin + 31) / 32 * 32;
    if (k2p > 256) return false;
    long mpix = (long)g.B * g.Ho * g.Wo;
    return mpix >= 256 && mpix % 32 == 0;
}
static cg_conv_geom patch_geom(const cg_conv_geom& g) {
    cg_conv_geom p = g;
    p.H = g.Ho; p.W = g.Wo; p.Cin = (g.KH * g.KW * g.Cin + 31) / 32 * 32;
    p.KH = p.KW = 1; p.stride = 1; p.pad = 0; p.ups = 0;
    return p;
}
static size_t patch_bytes(const cg_conv_geom& g) {
    cg_conv_geom p = patch_geom(g);
    return ((size_t)(g.x_groups == 1 ? 1 : g.G) * g.B * g.Ho * g.Wo * p.Cin * sizeof(float) + 1023) & ~(size_t)1023;
}
static size_t patch_w_bytes(const cg_conv_geom& g) {
    cg_conv_geom p = patch_geom(g);
    return ((size_t)g.G * g.Cout * p.Cin * sizeof(float) + 1023) & ~(size_t)1023;
}

__global__ void im2col_small_kernel(const float* __restrict__ x, float* __restrict__ P, long total4, int H, int W, int Cin, int Ho, int Wo,
                                    int KH, int KW, int stride, int pad, int K2, int K2p) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // one float4 slot of P
    if (i >= total4) return;
    int slots = K2p >> 2;
    int slot = (int)(i % slots);
    long pix = i / slots;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    int k = slot * 4;
    if (k < K2) {
        int tap = k / Cin, ci = k - tap * Cin;
        int kh = tap / KW, kw = tap - kh * KW;
        int ow = (int)(pix % Wo);
        long t = pix / Wo;
        int oh = (int)(t % Ho);
        long n = t / Ho;
        int ih = oh * stride - pad + kh, iw = ow * stride - pad + kw;
        if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = __ldg(reinterpret_cast<const float4*>(x + ((n * H + ih) * W + iw) * Cin + ci));
    }
    reinterpret_cast<float4*>(P)[i] = v;
}
// rows of K2 floats <-> rows of K2p floats (zero padded); dir 0: pad (w -> wp), 1: unpad (dwp -> dw)
__global__ void pad_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, long rows, int K2, int K2p, int dir) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (dir == 0) {
        if (i >= rows * K2p) return;
        long r = i / K2p;
        int k = (int)(i - r * K2p);
        dst[i] = k < K2 ? __ldg(src + r * K2 + k) : 0.f;
    } else {
        if (i >= rows * K2) return;
        long r = i / K2;
        int k = (int)(i - r * K2);
        dst[i] = __ldg(src + r * K2p + k);
    }
}
static int run_im2col(const cg_conv_geom& g, const float* x, float* P, cudaStream_t st) {
    cg_conv_geom p = patch_geom(g);
    long nimg = (long)(g.x_groups == 1 ? 1 : g.G) * g.B;
    long total4 = nimg * g.Ho * g.Wo * (p.Cin / 4);
    launch_k(im2col_small_kernel, cdiv(total4, 256), 256, 0, st, x, P, total4, g.H, g.W, g.Cin, g.Ho, g.Wo, g.KH, g.KW, g.stride, g.pad,
                                                          g.KH * g.KW * g.Cin, p.Cin);
    return check_launch("im2col_small");
}

}  // namespace cg

using namespace cg;

extern "C" const char* cg_last_error(void) { return g_err; }

extern "C" int cg_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        set_error("cudaGetDevice: %s", cudaGetErrorString(e));
        return CG_ERR_NO_DEVICE;
    }
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) {
        set_error("cudaGetDeviceProperties: %s", cudaGetErrorString(e));
        return CG_ERR_NO_DEVICE;
    }
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    return prop.multiProcessorCount;
}

extern "C" int cg_set_tensor_core_mode(int mode) {
    int prev = g_tc_mode;
    g_tc_mode = mode == 1 ? 7 : (mode & 7);  // 1 = everything; otherwise a bit mask: 1 forward, 2 data gradient, 4 weight gradient
    g_small_bn = ((mode >> 23) & 1) ? 0 : 1;  // bit 23: keep the widest N tile even when the launch has fewer tiles than SMs
    g_wgrad_tma = ((mode >> 25) & 1) ? 0 : 1;  // bit 25: stride-1 weight gradients on wgrad_tc_kernel instead of wgrad_tma_kernel
    g_pdl = (mode >> 22) & 1;  // bit 22: programmatic dependent launch
    g_tc_serial_epilogue = (mode >> 26) & 1;  // bit 26: conv_tc_kernel's previous epilogue and tile walk
    g_tc_reg_epilogue = (mode >> 27) & 1;  // bit 27: conv_tc_kernel's register epilogue everywhere (no shared-memory / TMA epilogue)
    return prev;
}

extern "C" uint64_t cg_launch_count(void) { return g_launches.load(); }
extern "C" void cg_tensor_map_cache_stats(uint64_t* hits, uint64_t* misses) { tc_map_cache_stats(hits, misses); }

extern "C" int cg_zero(void* ptr, size_t bytes, void* stream) {
    cudaError_t e = cudaMemsetAsync(ptr, 0, bytes, (cudaStream_t)stream);
    if (e != cudaSuccess) {
        set_error("cg_zero: %s", cudaGetErrorString(e));
        return CG_ERR_CUDA;
    }
    return CG_OK;
}

extern "C" size_t cg_conv_workspace_bytes(const cg_conv_geom* g, int which) {
    if (!g) return 0;
    ConvDims d = conv_dims(*g);
    size_t need = 0;
    // the same predicates as the dispatch in cg_conv_fwd / cg_conv_wgrad (the forward's activation is not known here: a tanh
    // layer falls through to the direct path, so the larger of the two needs is reported)
    const bool patch_fwd = which == 0 && (g_tc_mode & 1) && patch_path(*g) && g->KH * g->KW >= 16;
    if (which == 2 && small_wgrad_supported(*g)) return small_ws(*g, 2);
    if (which == 1 && small_dgrad_supported(*g)) return small_ws(*g, 1);
    const bool patch_wgrad = which == 2 && (g_tc_mode & 4) && patch_path(*g);
    if (patch_fwd || patch_wgrad) {
        cg_conv_geom p = patch_geom(*g);
        ConvDims dp = conv_dims(p);
        size_t inner = which == 2 ? tc_wgrad_ws(p) : 0;
        size_t cs = which == 2 ? colsum_ws(g->G, dp.Mpix, g->Cout) : 0;
        if (cs > inner) inner = cs;
        need = patch_bytes(*g) + 2 * patch_w_bytes(*g) + inner;
        if (which == 2) return need;
    }
    if (which == 0 && (g_tc_mode & 1) && tc_fwd_supported(*g)) { size_t t = tc_fwd_ws(*g); need = t > need ? t : need; }
    if (which == 1) {
        if (g->ups) need = (size_t)g->G * g->B * d.Hin * d.Win * g->Cin * sizeof(float);
        if ((g_tc_mode & 2) && tc_dgrad_supported(*g)) { size_t t = tc_dgrad_ws(*g); need = t > need ? t : need; }
    }
    if (which == 2) {
        size_t a = ((g_tc_mode & 4) && tc_wgrad_supported(*g)) ? tc_wgrad_ws(*g) : simt_wgrad_ws(*g);
        size_t b = colsum_ws(g->G, d.Mpix, g->Cout);
        need = a > b ? a : b;
    }
    return need;
}

extern "C" int cg_conv_fwd(const cg_conv_geom* g, const float* x, const float* w, const float* bias, float* y, int act,
                           float slope, void* ws, size_t ws_bytes, void* stream) {
    if (int rc = validate_geom(*g)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (small_fwd_supported(*g, act)) return small_conv_fwd(*g, x, w, bias, y, st);
    // forward: the patch matrix pays off when there are many taps (7x7: 49, 4x4: 16); the 3x3 pair layer is faster
    // straight through TMA im2col with 32-byte rows (9 taps: the patch matrix would be nearly as large as the map it replaces)
    if ((g_tc_mode & 1) && patch_path(*g) && g->KH * g->KW >= 16 && act != CG_ACT_TANH) {
        size_t need = cg_conv_workspace_bytes(g, 0);
        if (need > ws_bytes) {
            set_error("conv_fwd(patch path): workspace %zu < %zu bytes", ws_bytes, need);
            return CG_ERR_WORKSPACE;
        }
        cg_conv_geom p = patch_geom(*g);
        float* P = (float*)ws;
        float* wp = (float*)((uint8_t*)ws + patch_bytes(*g));
        if (int rc = run_im2col(*g, x, P, st)) return rc;
        long rows = (long)g->G * g->Cout;
        launch_k(pad_rows_kernel, cdiv(rows * p.Cin, 256), 256, 0, st, w, wp, rows, g->KH * g->KW * g->Cin, p.Cin, 0);
        if (int rc = check_launch("pad_rows")) return rc;
        return tc_conv_fwd(p, P, wp, bias, y, act, slope, nullptr, 0, st);
    }
    if ((g_tc_mode & 1) && tc_fwd_supported(*g) && !(act == CG_ACT_TANH && g->Cout > 16))
        return tc_conv_fwd(*g, x, w, bias, y, act, slope, ws, ws_bytes, st);
    return simt_conv_fwd(*g, x, w, bias, y, act, slope, st);
}

extern "C" int cg_conv_dgrad(const cg_conv_geom* g, const float* dy, const float* w, float* dx, const float* addend,
                             const float* mask_src, float mask_slope, void* ws, size_t ws_bytes, void* stream) {
    if (int rc = validate_geom(*g)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (small_dgrad_supported(*g)) return small_conv_dgrad(*g, dy, w, dx, addend, mask_src, mask_slope, ws, ws_bytes, st);
    if ((g_tc_mode & 2) && tc_dgrad_supported(*g)) return tc_conv_dgrad(*g, dy, w, dx, addend, mask_src, mask_slope, ws, ws_bytes, st);
    if (!g->ups) return simt_conv_dgrad(*g, dy, w, dx, addend, mask_src, mask_slope, st);
    size_t need = cg_conv_workspace_bytes(g, 1);
    if (need > ws_bytes) {
        set_error("conv_dgrad: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    if (int rc = simt_conv_dgrad(*g, dy, w, (float*)ws, nullptr, nullptr, 0.f, st)) return rc;
    return pool2x2_sum((const float*)ws, dx, addend, mask_src, mask_slope, (long)g->G * g->B, g->H, g->W, g->Cin, st);
}

extern "C" int cg_conv_wgrad(const cg_conv_geom* g, const float* x, const float* dy, float* dw, float* db, void* ws,
                             size_t ws_bytes, void* stream) {
    if (int rc = validate_geom(*g)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (small_wgrad_supported(*g)) return small_conv_wgrad(*g, x, dy, dw, db, ws, ws_bytes, st);
    if ((g_tc_mode & 4) && patch_path(*g)) {
        size_t need = cg_conv_workspace_bytes(g, 2);
        if (need > ws_bytes) {
            set_error("conv_wgrad(patch path): workspace %zu < %zu bytes", ws_bytes, need);
            return CG_ERR_WORKSPACE;
        }
        cg_conv_geom p = patch_geom(*g);
        ConvDims dp = conv_dims(p);
        float* P = (float*)ws;
        float* dwp = (float*)((uint8_t*)ws + patch_bytes(*g));
        uint8_t* inner = (uint8_t*)ws + patch_bytes(*g) + 2 * patch_w_bytes(*g);
        size_t inner_bytes = ws_bytes - (size_t)(inner - (uint8_t*)ws);
        if (int rc = run_im2col(*g, x, P, st)) return rc;
        if (int rc = tc_conv_wgrad(p, P, dy, dwp, inner, inner_bytes, st)) return rc;
        long rows = (long)g->G * g->Cout;
        int K2 = g->KH * g->KW * g->Cin;
        launch_k(pad_rows_kernel, cdiv(rows * K2, 256), 256, 0, st, dwp, dw, rows, K2, p.Cin, 1);
        if (int rc = check_launch("unpad_rows")) return rc;
        if (db) return colsum(dy, db, g->G, dp.Mpix, g->Cout, inner, inner_bytes, st);
        return CG_OK;
    }
    if ((g_tc_mode & 4) && tc_wgrad_supported(*g)) {
        if (int rc = tc_conv_wgrad(*g, x, dy, dw, ws, ws_bytes, st)) return rc;
    } else {
        if (int rc = simt_conv_wgrad(*g, x, dy, dw, ws, ws_bytes, st)) return rc;
    }
    if (db) {
        ConvDims d = conv_dims(*g);
        return colsum(dy, db, g->G, d.Mpix, g->Cout, ws, ws_bytes, st);
    }
    return CG_OK;
}

extern "C" int cg_upsample2x_bwd(const float* d_up, float* dx, int N, int H, int W, int C, void* stream) {
    CG_REQUIRE(C % 4 == 0, "upsample2x_bwd: C=%d must be a multiple of 4", C);
    return pool2x2_sum(d_up, dx, nullptr, nullptr, 0.f, N, H, W, C, (cudaStream_t)stream);
}

// Convolution (no bias, no activation) + instance-norm statistics of its output in one call: on the tensor path the
// per-channel sums are produced by the convolution epilogue (no second pass over y); otherwise conv then cg_in_stats.
extern "C" int cg_conv_fwd_stats(const cg_conv_geom* g, const float* x, const float* w, float* y, float* mean, float* rstd, float eps,
                                 void* ws, size_t ws_bytes, void* stream) {
    if (int rc = validate_geom(*g)) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    const int HW = g->Ho * g->Wo;
    int chunks = ((g_tc_mode & 1) && tc_fwd_supported(*g) && !patch_path(*g)) ? tc_fwd_stats_chunks(*g) : 0;
    if (chunks > 0) {
        long GBC = (long)g->G * g->B * g->Cout;
        size_t part_bytes = ((size_t)chunks * GBC * 2 * sizeof(float) + 1023) & ~(size_t)1023;
        size_t inner = tc_fwd_ws(*g);
        if (part_bytes + inner > ws_bytes) {
            set_error("conv_fwd_stats: workspace %zu < %zu bytes", ws_bytes, part_bytes + inner);
            return CG_ERR_WORKSPACE;
        }
        float* part = (float*)ws;
        if (int rc = tc_conv_fwd(*g, x, w, nullptr, y, CG_ACT_NONE, 0.f, (uint8_t*)ws + part_bytes, ws_bytes - part_bytes, st, part)) return rc;
        return in_stats_finalize(part, mean, rstd, GBC, chunks, HW, eps, st);
    }
    if (int rc = cg_conv_fwd(g, x, w, nullptr, y, CG_ACT_NONE, 0.f, ws, ws_bytes, stream)) return rc;
    return cg_in_stats(y, mean, rstd, g->G, g->B, HW, g->Cout, eps, ws, ws_bytes, stream);
}
extern "C" size_t cg_conv_fwd_stats_workspace_bytes(const cg_conv_geom* g) {
    if (!g) return 0;
    size_t a = cg_conv_workspace_bytes(g, 0);
    long GBC = (long)g->G * g->B * g->Cout;
    int chunks = ((g_tc_mode & 1) && tc_fwd_supported(*g) && !patch_path(*g)) ? tc_fwd_stats_chunks(*g) : 0;
    size_t fused = chunks > 0 ? (((size_t)chunks * GBC * 2 * sizeof(float) + 1023) & ~(size_t)1023) + tc_fwd_ws(*g) : 0;
    size_t plain = (size_t)(((long)g->Ho * g->Wo + 511) / 512) * GBC * 2 * sizeof(float);
    size_t m = a > fused ? a : fused;
    return m > plain ? m : plain;
}
