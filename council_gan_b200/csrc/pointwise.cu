// Image-space, loss and optimiser kernels (all HBM-bound; coalesced, vectorised where the layout allows).
#include "common.cuh"
#include "mask_head.cuh"

namespace cg {

__device__ __forceinline__ float4 f4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// block-wide sum of `n` floats per thread; result valid in thread 0
template <int N>
__device__ __forceinline__ void block_reduce(float (&v)[N], float* smem /* >= N*32 */) {
#pragma unroll
    for (int i = 0; i < N; i++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
    int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    __syncthreads();
    if (lane == 0)
#pragma unroll
        for (int i = 0; i < N; i++) smem[i * 32 + warp] = v[i];
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int i = 0; i < N; i++) {
            float t = lane < nw ? smem[i * 32 + lane] : 0.f;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
            v[i] = t;
        }
    }
}

// ---- attention-mask head: Decoder_V2_atten.forward networks.py:398-407 (compositing in mask_head.cuh) -----
__global__ void mask_head_fwd_kernel(const float* __restrict__ h, const float* __restrict__ x_in, float* __restrict__ x_fake,
                                     float* __restrict__ mask, long total, long per_group) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    MaskHeadPix p;
    mask_composite(h + i * 12, x_in + (i % per_group) * 4, p);
    reinterpret_cast<float4*>(x_fake)[i] = make_float4(p.im[3][0], p.im[3][1], p.im[3][2], 0.f);
    reinterpret_cast<float4*>(mask)[i] = make_float4(p.mk[0], p.mk[1], p.mk[2], 0.f);
}

__global__ void mask_head_bwd_kernel(const float* __restrict__ h, const float* __restrict__ x_in,
                                     const float* __restrict__ d_xfake, const float* __restrict__ d_mask,
                                     float* __restrict__ dh_pre, long total, long per_group) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    MaskHeadPix p;
    mask_composite(h + i * 12, x_in + (i % per_group) * 4, p);
    float4 dx = f4(d_xfake + i * 4);
    float dim[3] = {dx.x, dx.y, dx.z};
    float dm[3] = {0.f, 0.f, 0.f};
    if (d_mask) {
        float4 d = f4(d_mask + i * 4);
        dm[0] = d.x; dm[1] = d.y; dm[2] = d.z;
    }
    float out[12];
    mask_head_grad(p, dim, dm, out);
    store12(dh_pre + i * 12, out);
}

// ---- AvgPool2d(3, stride 2, pad 1, count_include_pad=False): networks.py:32,129 ------------------
__global__ void avgpool_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long total, int H, int W, int C4) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int Ho = H / 2, Wo = W / 2;
    int c = (int)(i % C4);
    long t = i / C4;
    int ow = (int)(t % Wo);
    t /= Wo;
    int oh = (int)(t % Ho);
    long n = t / Ho;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    int cnt = 0;
    for (int dh = -1; dh <= 1; dh++) {
        int ih = 2 * oh + dh;
        if (ih < 0 || ih >= H) continue;
        for (int dw = -1; dw <= 1; dw++) {
            int iw = 2 * ow + dw;
            if (iw < 0 || iw >= W) continue;
            float4 v = __ldg(reinterpret_cast<const float4*>(x) + ((n * H + ih) * W + iw) * C4 + c);
            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
            cnt++;
        }
    }
    float r = 1.f / (float)cnt;
    reinterpret_cast<float4*>(y)[i] = make_float4(s.x * r, s.y * r, s.z * r, s.w * r);
}

__device__ __forceinline__ int pool_cnt(int o, int L) {  // valid taps of output index o along one axis
    int c = 0;
    for (int d = -1; d <= 1; d++) {
        int i = 2 * o + d;
        c += (i >= 0 && i < L);
    }
    return c;
}
// one thread per input pixel; gathers from the <=2x2 output windows that cover it
__global__ void avgpool_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, long total, int H, int W, int Cy,
                                   int Cx, int nch, int accumulate) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int Ho = H / 2, Wo = W / 2;
    int iw = (int)(i % W);
    long t = i / W;
    int ih = (int)(t % H);
    long n = t / H;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    // outputs oh with |ih - 2*oh| <= 1
    for (int oh = (ih - 1 + 1) / 2; oh <= (ih + 1) / 2; oh++) {
        if (oh < 0 || oh >= Ho || abs(ih - 2 * oh) > 1) continue;
        int ch = pool_cnt(oh, H);
        for (int ow = iw / 2; ow <= (iw + 1) / 2; ow++) {
            if (ow < 0 || ow >= Wo || abs(iw - 2 * ow) > 1) continue;
            float r = 1.f / (float)(ch * pool_cnt(ow, W));
            const float* p = dy + ((n * Ho + oh) * Wo + ow) * Cy;
            for (int c = 0; c < nch; c++) acc[c] += __ldg(p + c) * r;
        }
    }
    float* o = dx + i * Cx;
    for (int c = 0; c < nch; c++) o[c] = accumulate ? o[c] + acc[c] : acc[c];
}

// style encoder tail (networks.py:348: nn.AdaptiveAvgPool2d(1)): one thread per (image, channel) sums its HW pixels in pixel order
__global__ void global_avgpool_fwd_kernel(const float* __restrict__ h, float* __restrict__ y, int N, int HW, int C) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)N * C) return;
    const long n = i / C;
    const int c = (int)(i - n * C);
    const float* p = h + n * HW * (long)C + c;
    float s = 0.f;
    for (int k = 0; k < HW; k++) s += __ldg(p + (long)k * C);
    y[i] = s / (float)HW;
}

// dh = dy / HW at every pixel, times the ReLU gate h > 0 when relu_gate (h: the pool's input, a ReLU output)
__global__ void global_avgpool_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ h, float* __restrict__ dh, long total4,
                                          int HW, int C4, int relu_gate) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total4) return;
    const long n = i / ((long)HW * C4);
    const int c = (int)(i % C4);
    const float r = 1.f / (float)HW;
    float4 g = __ldg(reinterpret_cast<const float4*>(dy) + n * C4 + c);
    g.x *= r; g.y *= r; g.z *= r; g.w *= r;
    if (relu_gate) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(h) + i);
        g.x = v.x > 0.f ? g.x : 0.f; g.y = v.y > 0.f ? g.y : 0.f; g.z = v.z > 0.f ? g.z : 0.f; g.w = v.w > 0.f ? g.w : 0.f;
    }
    reinterpret_cast<float4*>(dh)[i] = g;
}

__global__ void acc_slice_kernel(float* __restrict__ dst, const float* __restrict__ src, long npix, int Cd, int Cs, int nch) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    for (int c = 0; c < nch; c++) dst[i * Cd + c] += __ldg(src + i * Cs + c);
}

__global__ void gather_images_kernel(const float* __restrict__ pool0, int n0, const float* __restrict__ pool1,
                                     const int32_t* __restrict__ idx, const float* __restrict__ x_in, float* __restrict__ y,
                                     long total, int Bt, int B, int HW) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int pix = (int)(i % HW);
    long gn = i / HW;  // g*Bt + n
    int n = (int)(gn % Bt);
    int slot = __ldg(idx + gn);
    float4 v = slot < n0 ? f4(pool0 + ((long)slot * HW + pix) * 4) : f4(pool1 + ((long)(slot - n0) * HW + pix) * 4);
    if (x_in) {
        float4 u = f4(x_in + ((long)(n % B) * HW + pix) * 4);
        reinterpret_cast<float4*>(y)[i * 2] = v;
        reinterpret_cast<float4*>(y)[i * 2 + 1] = u;
    } else {
        reinterpret_cast<float4*>(y)[i] = v;
    }
}

// do_Dis_only_gray (trainer_council.py:736-737, 761, 765, 504, 510): torch.sum(x, 1) / input_dim on every live lane -- the sum in
// channel order, then a true division -- and 0 on lane 3
__global__ void gather_images_gray_kernel(const float* __restrict__ pool0, int n0, const float* __restrict__ pool1,
                                          const int32_t* __restrict__ idx, float* __restrict__ y, long total, int HW) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int pix = (int)(i % HW);
    int slot = __ldg(idx + i / HW);
    float4 v = slot < n0 ? f4(pool0 + ((long)slot * HW + pix) * 4) : f4(pool1 + ((long)(slot - n0) * HW + pix) * 4);
    float g = __fdiv_rn(v.x + v.y + v.z, 3.f);
    reinterpret_cast<float4*>(y)[i] = make_float4(g, g, g, 0.f);
}

// autograd of the conversion above: d x_c = g0/3 + g1/3 + g2/3 on every live lane (the division's gradient, then the repeat's sum)
__global__ void gray_fold_kernel(float* __restrict__ d, long npix) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    float4 v = reinterpret_cast<const float4*>(d)[i];
    float g = __fdiv_rn(v.x, 3.f) + __fdiv_rn(v.y, 3.f) + __fdiv_rn(v.z, 3.f);
    reinterpret_cast<float4*>(d)[i] = make_float4(g, g, g, v.w);
}

// useRandomDis (trainer_council.py:499-501): dst[g] = src[map[g]] in every member-major segment [G][n] of a parameter bank.  Blocks
// are dealt to the segments in proportion to their size (blk0[s] = first block of segment s), so no block idles.
constexpr int GM_THREADS = 256, GM_UNROLL = 4;
struct MemberGather {
    int map[CG_LOSS_MAX_G];
    int G, nseg;
    long off[CG_GATHER_MAX_SEG], n[CG_GATHER_MAX_SEG];  // floats: segment start, per-member length
    int blk0[CG_GATHER_MAX_SEG + 1];
};
__global__ void __launch_bounds__(GM_THREADS) gather_members_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                                    const MemberGather mg) {
    pdl_trigger();
    pdl_wait();
    int s = 0;
    while (s + 1 < mg.nseg && (int)blockIdx.x >= mg.blk0[s + 1]) s++;
    const long n = mg.n[s], off = mg.off[s];
    const bool vec = (n & 3) == 0;  // segment starts are 64-float aligned
    const long per = vec ? n / 4 : n, total = per * mg.G;
    const long base = (long)(blockIdx.x - mg.blk0[s]) * GM_THREADS * GM_UNROLL + threadIdx.x;
#pragma unroll
    for (int u = 0; u < GM_UNROLL; u++) {
        const long i = base + (long)u * GM_THREADS;
        if (i >= total) break;
        const long g = i / per, k = i - g * per;
        const long from = (long)mg.map[g] * per + k;
        if (vec)
            reinterpret_cast<float4*>(dst + off)[i] = __ldg(reinterpret_cast<const float4*>(src + off) + from);
        else
            dst[off + i] = __ldg(src + off + from);
    }
}

__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, float* __restrict__ y, long total, int C, int HW, int Cp) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // over N*HW
    if (i >= total) return;
    long n = i / HW;
    int pix = (int)(i - n * HW);
    for (int c = 0; c < Cp; c++) y[i * Cp + c] = c < C ? __ldg(x + (n * C + c) * HW + pix) : 0.f;
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ x, float* __restrict__ y, long total, int C, int HW, int Cp) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // over N*HW
    if (i >= total) return;
    long n = i / HW;
    int pix = (int)(i - n * HW);
    for (int c = 0; c < C; c++) y[(n * C + c) * HW + pix] = __ldg(x + i * Cp + c);
}

// ---- LSGAN: networks.py:64,90,166,194 -----------------------------------------------------------
__global__ void __launch_bounds__(256) lsgan_fwd_kernel(const float* __restrict__ out, const float* __restrict__ targets,
                                                        const float* __restrict__ weights, float* __restrict__ sums,
                                                        float* __restrict__ loss, int nseg, int n_per_seg, int accumulate) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sm[32];
    const int g = blockIdx.x;
    float total = 0.f;
    for (int seg = 0; seg < nseg; seg++) {
        float t = __ldg(targets + seg);
        const float* p = out + ((long)g * nseg + seg) * n_per_seg;
        float v[1] = {0.f};
        for (int i = threadIdx.x; i < n_per_seg; i += blockDim.x) {
            float d = __ldg(p + i) - t;
            v[0] += d * d;
        }
        block_reduce<1>(v, sm);
        if (threadIdx.x == 0) {
            sums[g * nseg + seg] = v[0];
            total += __ldg(weights + g * nseg + seg) * (v[0] / (float)n_per_seg);
        }
    }
    if (threadIdx.x == 0) loss[g] = accumulate ? loss[g] + total : total;
}
__global__ void lsgan_bwd_kernel(const float* __restrict__ out, const float* __restrict__ targets, const float* __restrict__ coef,
                                 float* __restrict__ dout, long total, int nseg, int n_per_seg) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int gs = (int)(i / n_per_seg);
    dout[i] = __ldg(coef + gs) * (__ldg(out + i) - __ldg(targets + gs % nseg));
}

// ---- focus losses: trainer_council.py:230-250 -----------------------------------------------------
constexpr int FC_PIX = 2048;  // pixels per block
__global__ void __launch_bounds__(256) focus_fwd_kernel(const float* __restrict__ mask, float* __restrict__ part, int B, int H,
                                                        int W, float center, float eps) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sm[4 * 32];
    const int g = blockIdx.y;
    const long npix = (long)B * H * W;
    const long p0 = (long)blockIdx.x * FC_PIX, p1 = min(npix, p0 + FC_PIX);
    const float* mb = mask + (long)g * npix * 4;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    for (long px = p0 + threadIdx.x; px < p1; px += blockDim.x) {
        int w = (int)(px % W);
        int h = (int)((px / W) % H);
        float4 m = f4(mb + px * 4);
        v[0] += 1.f / (fabsf(m.x - center) + eps) + 1.f / (fabsf(m.y - center) + eps) + 1.f / (fabsf(m.z - center) + eps);
        v[1] += m.x + m.y + m.z;
        if (h + 1 < H) {
            float4 d = f4(mb + (px + W) * 4);
            v[2] += fabsf(d.x - m.x) + fabsf(d.y - m.y) + fabsf(d.z - m.z);
        }
        if (w + 1 < W) {
            float4 r = f4(mb + (px + 1) * 4);
            v[3] += fabsf(r.x - m.x) + fabsf(r.y - m.y) + fabsf(r.z - m.z);
        }
    }
    block_reduce<4>(v, sm);
    if (threadIdx.x == 0) {
        float* o = part + ((long)blockIdx.x * gridDim.y + g) * 4;
        o[0] = v[0]; o[1] = v[1]; o[2] = v[2]; o[3] = v[3];
    }
}
__global__ void focus_final_kernel(const float* __restrict__ part, float* __restrict__ sums, int G4, int nchunks) {
    pdl_trigger();
    pdl_wait();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= G4) return;
    double s = 0.0;
    for (int k = 0; k < nchunks; k++) s += (double)part[(long)k * G4 + i];
    sums[i] = (float)s;
}
__device__ __forceinline__ float sgn(float x) { return (x > 0.f) - (x < 0.f); }
__global__ void focus_bwd_kernel(const float* __restrict__ mask, const float* __restrict__ coef, float* __restrict__ dmask,
                                 long total, long npix, int H, int W, float center, float eps) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // over G*npix
    if (i >= total) return;
    int g = (int)(i / npix);
    long px = i - (long)g * npix;
    int w = (int)(px % W);
    int h = (int)((px / W) % H);
    float c01 = __ldg(coef + g * 3), cs = __ldg(coef + g * 3 + 1), ctv = __ldg(coef + g * 3 + 2);
    const float* mp = mask + i * 4;
    float4 m = f4(mp);
    float mm[3] = {m.x, m.y, m.z}, o[3];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        float d = mm[c] - center;
        float den = fabsf(d) + eps;
        o[c] = cs - c01 * sgn(d) / (den * den);
    }
    if (ctv != 0.f) {
        float tv[3] = {0.f, 0.f, 0.f};
        if (h + 1 < H) { float4 q = f4(mp + (long)W * 4); tv[0] -= sgn(q.x - m.x); tv[1] -= sgn(q.y - m.y); tv[2] -= sgn(q.z - m.z); }
        if (h > 0)     { float4 q = f4(mp - (long)W * 4); tv[0] += sgn(m.x - q.x); tv[1] += sgn(m.y - q.y); tv[2] += sgn(m.z - q.z); }
        if (w + 1 < W) { float4 q = f4(mp + 4);           tv[0] -= sgn(q.x - m.x); tv[1] -= sgn(q.y - m.y); tv[2] -= sgn(q.z - m.z); }
        if (w > 0)     { float4 q = f4(mp - 4);           tv[0] += sgn(m.x - q.x); tv[1] += sgn(m.y - q.y); tv[2] += sgn(m.z - q.z); }
#pragma unroll
        for (int c = 0; c < 3; c++) o[c] += ctv * tv[c];
    }
    reinterpret_cast<float4*>(dmask)[i] = make_float4(o[0], o[1], o[2], 0.f);
}

// ---- Adam: torch.optim.Adam (trainer_council.py:170-179): L2 decay into the gradient, eps 1e-8 ----
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                            long n, float lr_c1, float b1, float b2, float eps, float wd, float rsq_c2, float gscale) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    long stride = (long)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        float pv = p[i];
        float gv = __ldg(g + i) * gscale + wd * pv;
        float mv = b1 * m[i] + (1.f - b1) * gv;
        float vv = b2 * v[i] + (1.f - b2) * gv * gv;
        m[i] = mv;
        v[i] = vv;
        float denom = sqrtf(vv) * rsq_c2 + eps;
        p[i] = pv - lr_c1 * (mv / denom);
    }
}

}  // namespace cg

using namespace cg;
#define ST ((cudaStream_t)stream)

extern "C" int cg_mask_head_fwd(const float* h, const float* x_in, float* x_fake, float* mask, int G, int B, int HW, void* stream) {
    long per = (long)B * HW, total = per * G;
    launch_k(mask_head_fwd_kernel, cdiv(total, 256), 256, 0, ST, h, x_in, x_fake, mask, total, per);
    return check_launch("mask_head_fwd");
}
extern "C" int cg_mask_head_bwd(const float* h, const float* x_in, const float* d_xfake, const float* d_mask, float* dh_pre,
                                int G, int B, int HW, void* stream) {
    long per = (long)B * HW, total = per * G;
    launch_k(mask_head_bwd_kernel, cdiv(total, 256), 256, 0, ST, h, x_in, d_xfake, d_mask, dh_pre, total, per);
    return check_launch("mask_head_bwd");
}
extern "C" int cg_avgpool_fwd(const float* x, float* y, int N, int H, int W, int C, void* stream) {
    CG_REQUIRE(C % 4 == 0 && H % 2 == 0 && W % 2 == 0, "avgpool_fwd: C=%d H=%d W=%d unsupported", C, H, W);
    long total = (long)N * (H / 2) * (W / 2) * (C / 4);
    launch_k(avgpool_fwd_kernel, cdiv(total, 256), 256, 0, ST, x, y, total, H, W, C / 4);
    return check_launch("avgpool_fwd");
}
extern "C" int cg_avgpool_bwd(const float* dy, float* dx, int N, int H, int W, int Cy, int Cx, int nch, int accumulate, void* stream) {
    CG_REQUIRE(nch <= 4 && nch <= Cy && nch <= Cx && H % 2 == 0 && W % 2 == 0, "avgpool_bwd: bad lanes/sizes");
    long total = (long)N * H * W;
    launch_k(avgpool_bwd_kernel, cdiv(total, 256), 256, 0, ST, dy, dx, total, H, W, Cy, Cx, nch, accumulate);
    return check_launch("avgpool_bwd");
}
extern "C" int cg_global_avgpool_fwd(const float* h, float* y, int N, int HW, int C, void* stream) {
    CG_REQUIRE(h && y && N >= 1 && HW >= 1 && C >= 1, "global_avgpool_fwd: N=%d HW=%d C=%d out of range", N, HW, C);
    launch_k(global_avgpool_fwd_kernel, cdiv((long)N * C, 256), 256, 0, ST, h, y, N, HW, C);
    return check_launch("global_avgpool_fwd");
}
extern "C" int cg_global_avgpool_bwd(const float* dy, const float* h, float* dh, int N, int HW, int C, int relu_gate, void* stream) {
    CG_REQUIRE(dy && dh && (h || !relu_gate) && N >= 1 && HW >= 1 && C >= 4 && C % 4 == 0,
               "global_avgpool_bwd: N=%d HW=%d C=%d out of range (C must be a multiple of 4)", N, HW, C);
    const long total4 = (long)N * HW * (C / 4);
    launch_k(global_avgpool_bwd_kernel, cdiv(total4, 256), 256, 0, ST, dy, h, dh, total4, HW, C / 4, relu_gate);
    return check_launch("global_avgpool_bwd");
}
extern "C" int cg_acc_slice(float* dst, const float* src, long npix, int Cd, int Cs, int nch, void* stream) {
    launch_k(acc_slice_kernel, cdiv(npix, 256), 256, 0, ST, dst, src, npix, Cd, Cs, nch);
    return check_launch("acc_slice");
}
extern "C" int cg_gather_images(const float* pool0, int n0, const float* pool1, const int32_t* idx, const float* x_in, float* y,
                                int G, int Bt, int B, int HW, void* stream) {
    long total = (long)G * Bt * HW;
    launch_k(gather_images_kernel, cdiv(total, 256), 256, 0, ST, pool0, n0, pool1, idx, x_in, y, total, Bt, B, HW);
    return check_launch("gather_images");
}
extern "C" int cg_gather_images_gray(const float* pool0, int n0, const float* pool1, const int32_t* idx, const float* x_in, float* y,
                                     int G, int Bt, int B, int HW, void* stream) {
    CG_REQUIRE(!x_in, "gather_images_gray: x_in must be NULL (the council discriminators see colour)");
    CG_REQUIRE(pool0 && idx && y && G >= 1 && Bt >= 1 && B >= 1 && HW >= 1, "gather_images_gray: G=%d Bt=%d HW=%d out of range", G,
               Bt, HW);
    long total = (long)G * Bt * HW;
    launch_k(gather_images_gray_kernel, cdiv(total, 256), 256, 0, ST, pool0, n0, pool1, idx, y, total, HW);
    return check_launch("gather_images_gray");
}
extern "C" int cg_gray_fold(float* d_x, long npix, void* stream) {
    CG_REQUIRE(d_x && npix >= 1, "gray_fold: npix=%ld out of range", npix);
    launch_k(gray_fold_kernel, cdiv(npix, 256), 256, 0, ST, d_x, npix);
    return check_launch("gray_fold");
}
extern "C" int cg_gather_members(const float* src, float* dst, const int64_t* host_off, const int64_t* host_n, int nseg,
                                 const int32_t* host_map, int G, void* stream) {
    CG_REQUIRE(src && dst && host_off && host_n && host_map, "gather_members: NULL argument");
    CG_REQUIRE(G >= 1 && G <= CG_LOSS_MAX_G, "gather_members: G=%d out of range (1..%d)", G, CG_LOSS_MAX_G);
    CG_REQUIRE(nseg >= 1 && nseg <= CG_GATHER_MAX_SEG, "gather_members: nseg=%d out of range (1..%d)", nseg, CG_GATHER_MAX_SEG);
    MemberGather mg;
    mg.G = G;
    mg.nseg = nseg;
    for (int g = 0; g < G; g++) {
        CG_REQUIRE(host_map[g] >= 0 && host_map[g] < G, "gather_members: map[%d] = %d is not a member", g, host_map[g]);
        mg.map[g] = host_map[g];
    }
    long blocks = 0;
    for (int s = 0; s < nseg; s++) {
        CG_REQUIRE(host_off[s] >= 0 && host_n[s] >= 1, "gather_members: segment %d (off %lld, n %lld) out of range", s,
                   (long long)host_off[s], (long long)host_n[s]);
        CG_REQUIRE(host_off[s] % 4 == 0, "gather_members: segment %d starts at %lld, not a multiple of 4 floats", s,
                   (long long)host_off[s]);
        mg.off[s] = host_off[s];
        mg.n[s] = host_n[s];
        mg.blk0[s] = (int)blocks;
        const long per = host_n[s] % 4 == 0 ? host_n[s] / 4 : host_n[s];
        blocks += cdiv(per * G, (long)GM_THREADS * GM_UNROLL);
        CG_REQUIRE(blocks < (1L << 31), "gather_members: too many blocks");
    }
    mg.blk0[nseg] = (int)blocks;
    launch_k(gather_members_kernel, (int)blocks, GM_THREADS, 0, ST, src, dst, mg);
    return check_launch("gather_members");
}
extern "C" int cg_nchw_to_nhwc(const float* x, float* y, int N, int C, int HW, int Cp, void* stream) {
    long total = (long)N * HW;
    launch_k(nchw_to_nhwc_kernel, cdiv(total, 256), 256, 0, ST, x, y, total, C, HW, Cp);
    return check_launch("nchw_to_nhwc");
}
extern "C" int cg_nhwc_to_nchw(const float* x, float* y, int N, int C, int HW, int Cp, void* stream) {
    long total = (long)N * HW;
    launch_k(nhwc_to_nchw_kernel, cdiv(total, 256), 256, 0, ST, x, y, total, C, HW, Cp);
    return check_launch("nhwc_to_nchw");
}
extern "C" int cg_lsgan_fwd(const float* out, const float* targets, const float* weights, float* sums, float* loss, int G,
                            int nseg, int n_per_seg, int accumulate, void* stream) {
    launch_k(lsgan_fwd_kernel, G, 256, 0, ST, out, targets, weights, sums, loss, nseg, n_per_seg, accumulate);
    return check_launch("lsgan_fwd");
}
extern "C" int cg_lsgan_bwd(const float* out, const float* targets, const float* coef, float* dout, int G, int nseg, int n_per_seg,
                            void* stream) {
    long total = (long)G * nseg * n_per_seg;
    launch_k(lsgan_bwd_kernel, cdiv(total, 256), 256, 0, ST, out, targets, coef, dout, total, nseg, n_per_seg);
    return check_launch("lsgan_bwd");
}
extern "C" int cg_focus_fwd(const float* mask, float* sums, int G, int B, int H, int W, float center, float eps, void* ws,
                            size_t ws_bytes, void* stream) {
    long npix = (long)B * H * W;
    int nchunks = cdiv(npix, FC_PIX);
    size_t need = (size_t)nchunks * G * 4 * sizeof(float);
    if (need > ws_bytes) {
        set_error("focus_fwd: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    launch_k(focus_fwd_kernel, dim3(nchunks, G), 256, 0, ST, mask, (float*)ws, B, H, W, center, eps);
    if (int rc = check_launch("focus_fwd")) return rc;
    launch_k(focus_final_kernel, cdiv(G * 4, 64), 64, 0, ST, (const float*)ws, sums, G * 4, nchunks);
    return check_launch("focus_final");
}
extern "C" int cg_focus_bwd(const float* mask, const float* coef, float* dmask, int G, int B, int H, int W, float center,
                            float eps, void* stream) {
    long npix = (long)B * H * W, total = npix * G;
    launch_k(focus_bwd_kernel, cdiv(total, 256), 256, 0, ST, mask, coef, dmask, total, npix, H, W, center, eps);
    return check_launch("focus_bwd");
}
extern "C" int cg_adam_step(float* p, const float* g, float* m, float* v, long n, float lr, float beta1, float beta2, float eps,
                            float weight_decay, int step, float grad_scale, void* stream) {
    double bc1 = 1.0 - pow((double)beta1, step), bc2 = 1.0 - pow((double)beta2, step);
    float lr_c1 = (float)((double)lr / bc1), rsq_c2 = (float)(1.0 / sqrt(bc2));
    int blocks = cdiv(n, 256);
    const int cap = 16 * (tc_sm_count() > 0 ? tc_sm_count() : 1);
    if (blocks > cap) blocks = cap;
    launch_k(adam_kernel, blocks, 256, 0, ST, p, g, m, v, n, lr_c1, beta1, beta2, eps, weight_decay, rsq_c2, grad_scale);
    return check_launch("adam");
}
