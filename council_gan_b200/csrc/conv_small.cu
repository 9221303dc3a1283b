// Degenerate "convolutions" of the training step that are really vector operations, as exact-fp32 streaming kernels:
//
//   * the 512 -> 1 patch heads of MsImageDis / MsImageDisCouncil (nn.Conv2d(dim, 1, 1, 1, 0), networks.py:45,143):
//       forward   y[px]     = <x[px][:], w> + b              one warp per pixel
//       dgrad     dx[px][c] = dy[px] * w[c]  (* LeakyReLU')   one float4 per thread
//       wgrad     dw[c]     = sum_px dy[px] * x[px][c],  db = sum_px dy[px]     two-phase, fixed order
//   * the data gradient of the last MLP layer (nn.Linear(256, 5888), networks.py:438): an 8 x 5888 x 256 product per member
//
// The generic 64x64x16 SIMT tiles fit them badly (N = 1 wastes 63/64 of a tile; the MLP gradient has 5888-long reductions and
// 8 rows).  They are HBM-trivial: 67 MB at the largest call.
#include "common.cuh"

namespace cg {

__device__ __forceinline__ float4 s_ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// ---- Cout == 1 head: forward ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) head1_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                                        float* __restrict__ y, long npix, int C) {
    pdl_trigger();
    pdl_wait();
    const int g = blockIdx.y;
    const long px = (long)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (px >= npix) return;
    const int lane = threadIdx.x & 31;
    const float* xp = x + ((long)g * npix + px) * C;
    const float* wp = w + (long)g * C;
    float acc = 0.f;
    for (int c = lane * 4; c < C; c += 128) {
        float4 a = s_ld4(xp + c), b = s_ld4(wp + c);
        acc = fmaf(a.x, b.x, acc); acc = fmaf(a.y, b.y, acc); acc = fmaf(a.z, b.z, acc); acc = fmaf(a.w, b.w, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) y[(long)g * npix + px] = acc + (bias ? __ldg(bias + g) : 0.f);
}

// ---- Cout == 1 head: data gradient ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) head1_dgrad_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ dx,
                                                          const float* __restrict__ addend, const float* __restrict__ mask_src, float slope,
                                                          long npix, int C4) {
    pdl_trigger();
    pdl_wait();
    const int g = blockIdx.y;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // over npix * C4
    if (i >= npix * C4) return;
    const long px = i / C4;
    const int c4 = (int)(i - px * C4);
    const float d = __ldg(dy + (long)g * npix + px);
    const float4 ww = s_ld4(w + ((long)g * C4 + c4) * 4);
    float4 o = make_float4(d * ww.x, d * ww.y, d * ww.z, d * ww.w);
    const long off = ((long)g * npix * C4 + i) * 4;
    if (addend) {
        float4 a = s_ld4(addend + off);
        o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w;
    }
    if (mask_src) {
        float4 m = s_ld4(mask_src + off);
        o.x *= m.x > 0.f ? 1.f : slope; o.y *= m.y > 0.f ? 1.f : slope; o.z *= m.z > 0.f ? 1.f : slope; o.w *= m.w > 0.f ? 1.f : slope;
    }
    *reinterpret_cast<float4*>(dx + off) = o;
}

// ---- Cout == 1 head: weight + bias gradient ------------------------------------------------------------------------------
constexpr int H1_ROWS = 256;  // pixels per block
// part[chunk][g][C + 4]: columns 0..C-1 = sum dy*x, column C = sum dy
__global__ void __launch_bounds__(256) head1_wgrad_partial_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ part,
                                                                  long npix, int C) {
    pdl_trigger();
    pdl_wait();
    __shared__ float4 sm[256];
    __shared__ float sdy[8];
    const int g = blockIdx.y, chunk = blockIdx.x;
    const int lanes = C >> 2;               // threads across the channel axis (C = 512 -> 128)
    const int rowl = 256 / lanes;
    const int lane = threadIdx.x % lanes, rl = threadIdx.x / lanes;
    const long r0 = (long)chunk * H1_ROWS, r1 = min(npix, r0 + H1_ROWS);
    const float* xb = x + (long)g * npix * C + lane * 4;
    const float* db = dy + (long)g * npix;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    float sd = 0.f;
    if (rl < rowl)
        for (long r = r0 + rl; r < r1; r += rowl) {
            const float d = __ldg(db + r);
            const float4 v = s_ld4(xb + r * C);
            s.x = fmaf(d, v.x, s.x); s.y = fmaf(d, v.y, s.y); s.z = fmaf(d, v.z, s.z); s.w = fmaf(d, v.w, s.w);
            if (lane == 0) sd += d;
        }
    sm[threadIdx.x] = s;
    if (lane == 0 && rl < 8) sdy[rl] = sd;
    __syncthreads();
    if (rl == 0) {
        for (int k = 1; k < rowl; k++) {
            float4 a = sm[k * lanes + lane];
            s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
        }
        float* o = part + ((long)chunk * gridDim.y + g) * (C + 4);
        *reinterpret_cast<float4*>(o + lane * 4) = s;
        if (lane == 0) {
            float t = 0.f;
            for (int k = 0; k < rowl && k < 8; k++) t += sdy[k];
            o[C] = t;
        }
    }
}
__global__ void head1_wgrad_final_kernel(const float* __restrict__ part, float* __restrict__ dw, float* __restrict__ db, int G, int C, int nchunks) {
    pdl_trigger();
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;  // over G * (C + 1)
    if (i >= G * (C + 1)) return;
    const int g = i / (C + 1), c = i - g * (C + 1);
    double s = 0.0;
    for (int k = 0; k < nchunks; k++) s += (double)part[((long)k * G + g) * (C + 4) + c];
    if (c < C) dw[(long)g * C + c] = (float)s;
    else if (db) db[g] = (float)s;
}

// ---- data gradient of a wide linear layer on a 1x1 map: dx[g][b][ci] = sum_co dy[g][b][co] * w[g][co][ci] ------------------------
constexpr int LD_SLICE = 64;  // output channels (reduction index) per block
constexpr int LD_MAXB = 16;
// part[slice][g][b][Cin]
__global__ void __launch_bounds__(256) lin_dgrad_partial_kernel(const float* __restrict__ dy, const float* __restrict__ w, float* __restrict__ part,
                                                                int B, int Cin, int Cout) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sdy[LD_MAXB][LD_SLICE];
    const int g = blockIdx.y, slice = blockIdx.x;
    const int co0 = slice * LD_SLICE, n = min(LD_SLICE, Cout - co0);
    for (int i = threadIdx.x; i < B * LD_SLICE; i += blockDim.x) {
        const int b = i / LD_SLICE, j = i - b * LD_SLICE;
        sdy[b][j] = j < n ? __ldg(dy + ((long)g * B + b) * Cout + co0 + j) : 0.f;
    }
    __syncthreads();
    for (int ci = threadIdx.x; ci < Cin; ci += blockDim.x) {
        float acc[LD_MAXB];
#pragma unroll
        for (int b = 0; b < LD_MAXB; b++) acc[b] = 0.f;
        const float* wp = w + ((long)g * Cout + co0) * Cin + ci;
        for (int j = 0; j < n; j++) {
            const float wv = __ldg(wp + (long)j * Cin);
#pragma unroll
            for (int b = 0; b < LD_MAXB; b++)
                if (b < B) acc[b] = fmaf(sdy[b][j], wv, acc[b]);
        }
#pragma unroll
        for (int b = 0; b < LD_MAXB; b++)
            if (b < B) part[(((long)slice * gridDim.y + g) * B + b) * Cin + ci] = acc[b];
    }
}
__global__ void lin_dgrad_final_kernel(const float* __restrict__ part, float* __restrict__ dx, const float* __restrict__ addend,
                                       const float* __restrict__ mask_src, float slope, long total, int nslices) {
    pdl_trigger();
    pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // over G * B * Cin
    if (i >= total) return;
    float s = 0.f;
    for (int k = 0; k < nslices; k++) s += __ldg(part + (long)k * total + i);
    if (addend) s += __ldg(addend + i);
    if (mask_src) s *= __ldg(mask_src + i) > 0.f ? 1.f : slope;
    dx[i] = s;
}

// ---- host ----------------------------------------------------------------------------------------------------------------
static bool is_head1(const cg_conv_geom& g) {
    return g.Cout == 1 && g.KH == 1 && g.KW == 1 && g.stride == 1 && g.pad == 0 && !g.ups && g.x_groups == g.G && g.Cin % 128 == 0 &&
           g.Cin <= 1024;
}
bool small_fwd_supported(const cg_conv_geom& g, int act) { return is_head1(g) && act == CG_ACT_NONE; }
bool small_dgrad_supported(const cg_conv_geom& g) {
    if (is_head1(g)) return true;
    // wide linear layer on a 1x1 map (the MLP's 256 -> 5888 output layer)
    return g.H == 1 && g.W == 1 && g.KH == 1 && g.KW == 1 && g.stride == 1 && g.pad == 0 && !g.ups && g.B <= LD_MAXB && g.Cout >= 1024;
}
bool small_wgrad_supported(const cg_conv_geom& g) { return is_head1(g); }

size_t small_ws(const cg_conv_geom& g, int which) {
    if (which == 2 && is_head1(g)) return (size_t)cdiv((long)g.B * g.H * g.W, H1_ROWS) * g.G * (g.Cin + 4) * sizeof(float);
    if (which == 1 && !is_head1(g) && small_dgrad_supported(g)) return (size_t)cdiv(g.Cout, LD_SLICE) * g.G * g.B * g.Cin * sizeof(float);
    return 0;
}

int small_conv_fwd(const cg_conv_geom& g, const float* x, const float* w, const float* bias, float* y, cudaStream_t st) {
    const long npix = (long)g.B * g.H * g.W;
    launch_k(head1_fwd_kernel, dim3(cdiv(npix, 8), g.G), 256, 0, st, x, w, bias, y, npix, g.Cin);
    return check_launch("head1_fwd");
}

int small_conv_dgrad(const cg_conv_geom& g, const float* dy, const float* w, float* dx, const float* addend, const float* mask_src,
                     float slope, void* ws, size_t ws_bytes, cudaStream_t st) {
    if (is_head1(g)) {
        const long npix = (long)g.B * g.H * g.W;
        const int C4 = g.Cin / 4;
        launch_k(head1_dgrad_kernel, dim3(cdiv(npix * C4, 256), g.G), 256, 0, st, dy, w, dx, addend, mask_src, slope, npix, C4);
        return check_launch("head1_dgrad");
    }
    size_t need = small_ws(g, 1);
    if (need > ws_bytes) {
        set_error("conv_dgrad(linear): workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    const int nsl = cdiv(g.Cout, LD_SLICE);
    launch_k(lin_dgrad_partial_kernel, dim3(nsl, g.G), 256, 0, st, dy, w, (float*)ws, g.B, g.Cin, g.Cout);
    if (int rc = check_launch("lin_dgrad_partial")) return rc;
    const long total = (long)g.G * g.B * g.Cin;
    launch_k(lin_dgrad_final_kernel, cdiv(total, 256), 256, 0, st, (const float*)ws, dx, addend, mask_src, slope, total, nsl);
    return check_launch("lin_dgrad_final");
}

int small_conv_wgrad(const cg_conv_geom& g, const float* x, const float* dy, float* dw, float* db, void* ws, size_t ws_bytes, cudaStream_t st) {
    size_t need = small_ws(g, 2);
    if (need > ws_bytes) {
        set_error("conv_wgrad(head): workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    const long npix = (long)g.B * g.H * g.W;
    const int nchunks = cdiv(npix, H1_ROWS);
    launch_k(head1_wgrad_partial_kernel, dim3(nchunks, g.G), 256, 0, st, x, dy, (float*)ws, npix, g.Cin);
    if (int rc = check_launch("head1_wgrad_partial")) return rc;
    launch_k(head1_wgrad_final_kernel, cdiv(g.G * (g.Cin + 1), 256), 256, 0, st, (const float*)ws, dw, db, g.G, g.Cin, nchunks);
    return check_launch("head1_wgrad_final");
}

}  // namespace cg
