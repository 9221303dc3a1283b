// SIMT fp32 implicit-GEMM convolutions: forward, data gradient, weight gradient.
//
// These are the exact-fp32 kernels of the library.  They serve (a) the layers that do not qualify
// for the tensor-core path (maps with < 128 pixels per member, the small MLP layers), (b) as the on-device
// reference the tensor-core kernels are verified against (cg_set_tensor_core_mode(0)).
//
// Reference call sites replaced: nn.Conv2d forward (networks.py:513,516) and its autograd
// (cuDNN dgrad / wgrad, reached from .backward() at trainer_council.py:633,779,882).
//
// Layouts: x[Gx][B][H][W][Cin], w[G][Cout][KH][KW][Cin], y[G][B][Ho][Wo][Cout]; GEMM view
//   fwd  : M = B*Ho*Wo pixels, N = Cout, K = (kh,kw,ci)
//   dgrad: M = input pixels of one stride-parity class, N = Cin, K = (kh',kw',co)
//   wgrad: M = Cout, N = (kh,kw,ci), K = pixels  (deterministic split-K)
#include "common.cuh"

namespace cg {

constexpr int BM = 64, BN = 64, BK = 16, NT = 256, SPAD = 4;

struct ConvKP {
    const float* x; const float* w; const float* bias; float* y;
    const float* addend; const float* mask_src;
    long xg;           // x group stride in floats (0: shared)
    int G, B, H, W, Cin, Ho, Wo, Cout, KH, KW, stride, pad, ups, Hin, Win;
    long Mpix; int Ktot;
    int act; float slope;
    // wgrad split-K
    int splits; long chunk;
};

static ConvKP make_kp(const cg_conv_geom& g) {
    ConvKP p{};
    ConvDims d = conv_dims(g);
    p.G = g.G; p.B = g.B; p.H = g.H; p.W = g.W; p.Cin = g.Cin; p.Ho = g.Ho; p.Wo = g.Wo; p.Cout = g.Cout;
    p.KH = g.KH; p.KW = g.KW; p.stride = g.stride; p.pad = g.pad; p.ups = g.ups;
    p.Hin = d.Hin; p.Win = d.Win; p.Mpix = d.Mpix; p.Ktot = d.Ktot;
    p.xg = g.x_groups == 1 ? 0 : (long)g.B * g.H * g.W * g.Cin;
    return p;
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// ------------------------------------------------------------------------------------------------
// forward
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) conv_fwd_simt_kernel(ConvKP p) {
    pdl_trigger();
    pdl_wait();
    __shared__ __align__(16) float As[BK][BM + SPAD];
    __shared__ __align__(16) float Bs[BK][BN + SPAD];
    const int tid = threadIdx.x;
    const int g = blockIdx.z;
    const long m0 = (long)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    const int lrow = tid >> 2, lkq = tid & 3;
    const int ty = tid >> 4, tx = tid & 15;

    // per-thread A row
    const long m = m0 + lrow;
    const bool mvalid = m < p.Mpix;
    int ih0 = 0, iw0 = 0;
    const float* xb = p.x + (long)g * p.xg;
    if (mvalid) {
        int hw = p.Ho * p.Wo;
        int b = (int)(m / hw);
        int r = (int)(m - (long)b * hw);
        int oh = r / p.Wo, ow = r - oh * p.Wo;
        ih0 = oh * p.stride - p.pad;
        iw0 = ow * p.stride - p.pad;
        xb += (long)b * p.H * p.W * p.Cin;
    }
    const int nB = n0 + lrow;
    const bool nvalid = nB < p.Cout;
    const float* wb = p.w + ((long)g * p.Cout + nB) * p.Ktot;

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.f;

    const int nk = (p.Ktot + BK - 1) / BK;
    float4 ra, rb;
    auto load = [&](int kt) {
        int k = kt * BK + lkq * 4;
        ra = make_float4(0.f, 0.f, 0.f, 0.f);
        rb = ra;
        if (k < p.Ktot) {
            if (mvalid) {
                int tap = k / p.Cin;
                int ci = k - tap * p.Cin;
                int kh = tap / p.KW, kw = tap - kh * p.KW;
                int ih = ih0 + kh, iw = iw0 + kw;
                if (ih >= 0 && ih < p.Hin && iw >= 0 && iw < p.Win) {
                    if (p.ups) { ih >>= 1; iw >>= 1; }
                    ra = ldg4(xb + ((long)ih * p.W + iw) * p.Cin + ci);
                }
            }
            if (nvalid) rb = ldg4(wb + k);
        }
    };
    auto store = [&]() {
        As[lkq * 4 + 0][lrow] = ra.x; As[lkq * 4 + 1][lrow] = ra.y;
        As[lkq * 4 + 2][lrow] = ra.z; As[lkq * 4 + 3][lrow] = ra.w;
        Bs[lkq * 4 + 0][lrow] = rb.x; Bs[lkq * 4 + 1][lrow] = rb.y;
        Bs[lkq * 4 + 2][lrow] = rb.z; Bs[lkq * 4 + 3][lrow] = rb.w;
    };
    load(0);
    store();
    __syncthreads();
    for (int kt = 0; kt < nk; kt++) {
        if (kt + 1 < nk) load(kt + 1);
#pragma unroll
        for (int kk = 0; kk < BK; kk++) {
            float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
        if (kt + 1 < nk) {
            store();
            __syncthreads();
        }
    }
    // epilogue
    const int n = n0 + tx * 4;
    float bv[4] = {0.f, 0.f, 0.f, 0.f};
    if (p.bias) {
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (n + j < p.Cout) bv[j] = __ldg(p.bias + (long)g * p.Cout + n + j);
    }
    const bool vec = (p.Cout & 3) == 0 && n + 3 < p.Cout;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        long mm = m0 + ty * 4 + i;
        if (mm >= p.Mpix) continue;
        float* yp = p.y + ((long)g * p.Mpix + mm) * p.Cout + n;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; j++) v[j] = apply_act(acc[i][j] + bv[j], p.act, p.slope);
        if (vec) {
            *reinterpret_cast<float4*>(yp) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; j++)
                if (n + j < p.Cout) yp[j] = v[j];
        }
    }
}

int simt_conv_fwd(const cg_conv_geom& g, const float* x, const float* w, const float* bias, float* y,
                  int act, float slope, cudaStream_t st) {
    ConvKP p = make_kp(g);
    p.x = x; p.w = w; p.bias = bias; p.y = y; p.act = act; p.slope = slope;
    dim3 grid(cdiv(p.Mpix, BM), cdiv(p.Cout, BN), p.G);
    launch_k(conv_fwd_simt_kernel, grid, NT, 0, st, p);
    return check_launch("conv_fwd_simt");
}

// ------------------------------------------------------------------------------------------------
// data gradient (w.r.t. the tensor the convolution sees: [G][B][Hin][Win][Cin])
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) conv_dgrad_simt_kernel(ConvKP p) {
    pdl_trigger();
    pdl_wait();
    __shared__ __align__(16) float As[BK][BM + SPAD];
    __shared__ __align__(16) float Bs[BK][BN + SPAD];
    const int tid = threadIdx.x;
    const int s = p.stride;
    const int ncls = s * s;
    const int g = blockIdx.z / ncls;
    const int cls = blockIdx.z - g * ncls;
    const int ph = cls / s, pw = cls - ph * s;
    const int ihf = ((ph - p.pad) % s + s) % s;
    const int iwf = ((pw - p.pad) % s + s) % s;
    const int Hc = p.Hin > ihf ? (p.Hin - ihf + s - 1) / s : 0;
    const int Wc = p.Win > iwf ? (p.Win - iwf + s - 1) / s : 0;
    const long Mc = (long)p.B * Hc * Wc;
    const long m0 = (long)blockIdx.x * BM;
    if (m0 >= Mc) return;
    const int n0 = blockIdx.y * BN;
    const int TH = p.KH / s, TW = p.KW / s;
    const int Kd = TH * TW * p.Cout;
    const int lrow = tid >> 2, lkq = tid & 3;
    const int ty = tid >> 4, tx = tid & 15;
    const int bkk = tid >> 4, bnq = tid & 15;

    const long m = m0 + lrow;
    const bool mvalid = m < Mc;
    int ihp = 0, iwp = 0;  // ih + pad, iw + pad
    const float* dyb = p.x + (long)g * p.Mpix * p.Cout;  // p.x carries dy here
    if (mvalid) {
        int hw = Hc * Wc;
        int b = (int)(m / hw);
        int r = (int)(m - (long)b * hw);
        int i = r / Wc, j = r - i * Wc;
        ihp = ihf + s * i + p.pad;
        iwp = iwf + s * j + p.pad;
        dyb += (long)b * p.Ho * p.Wo * p.Cout;
    }
    const int nB = n0 + bnq * 4;
    const bool nvalid = nB < p.Cin;
    const bool vecA = (p.Cout & 3) == 0;

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.f;

    const int nk = (Kd + BK - 1) / BK;
    float4 ra, rb;
    auto loadA1 = [&](int k) -> float {
        if (k >= Kd || !mvalid) return 0.f;
        int t = k / p.Cout;
        int co = k - t * p.Cout;
        int th = t / TW, tw = t - th * TW;
        int ohn = ihp - (ph + s * th), own = iwp - (pw + s * tw);
        if (ohn < 0 || own < 0) return 0.f;
        int oh = ohn / s, ow = own / s;
        if (oh >= p.Ho || ow >= p.Wo) return 0.f;
        return __ldg(dyb + ((long)oh * p.Wo + ow) * p.Cout + co);
    };
    auto load = [&](int kt) {
        int k = kt * BK + lkq * 4;
        ra = make_float4(0.f, 0.f, 0.f, 0.f);
        rb = ra;
        if (vecA) {
            if (k < Kd && mvalid) {
                int t = k / p.Cout;
                int co = k - t * p.Cout;
                int th = t / TW, tw = t - th * TW;
                int ohn = ihp - (ph + s * th), own = iwp - (pw + s * tw);
                if (ohn >= 0 && own >= 0) {
                    int oh = ohn / s, ow = own / s;
                    if (oh < p.Ho && ow < p.Wo) ra = ldg4(dyb + ((long)oh * p.Wo + ow) * p.Cout + co);
                }
            }
        } else {
            ra.x = loadA1(k); ra.y = loadA1(k + 1); ra.z = loadA1(k + 2); ra.w = loadA1(k + 3);
        }
        int kb = kt * BK + bkk;
        if (kb < Kd && nvalid) {
            int t = kb / p.Cout;
            int co = kb - t * p.Cout;
            int th = t / TW, tw = t - th * TW;
            int kh = ph + s * th, kw = pw + s * tw;
            rb = ldg4(p.w + (((long)g * p.Cout + co) * p.KH * p.KW + kh * p.KW + kw) * p.Cin + nB);
        }
    };
    auto store = [&]() {
        As[lkq * 4 + 0][lrow] = ra.x; As[lkq * 4 + 1][lrow] = ra.y;
        As[lkq * 4 + 2][lrow] = ra.z; As[lkq * 4 + 3][lrow] = ra.w;
        *reinterpret_cast<float4*>(&Bs[bkk][bnq * 4]) = rb;
    };
    load(0);
    store();
    __syncthreads();
    for (int kt = 0; kt < nk; kt++) {
        if (kt + 1 < nk) load(kt + 1);
#pragma unroll
        for (int kk = 0; kk < BK; kk++) {
            float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
            float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
        if (kt + 1 < nk) {
            store();
            __syncthreads();
        }
    }
    const int n = n0 + tx * 4;
    if (n >= p.Cin) return;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        long mm = m0 + ty * 4 + i;
        if (mm >= Mc) continue;
        int hw = Hc * Wc;
        int b = (int)(mm / hw);
        int r = (int)(mm - (long)b * hw);
        int ii = r / Wc, jj = r - ii * Wc;
        int ih = ihf + s * ii, iw = iwf + s * jj;
        long idx = ((((long)g * p.B + b) * p.Hin + ih) * p.Win + iw) * p.Cin + n;
        float4 v = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
        if (p.addend) {
            float4 a = ldg4(p.addend + idx);
            v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
        }
        if (p.mask_src) {
            float4 a = ldg4(p.mask_src + idx);
            v.x *= a.x > 0.f ? 1.f : p.slope; v.y *= a.y > 0.f ? 1.f : p.slope;
            v.z *= a.z > 0.f ? 1.f : p.slope; v.w *= a.w > 0.f ? 1.f : p.slope;
        }
        *reinterpret_cast<float4*>(p.y + idx) = v;
    }
}

int simt_conv_dgrad(const cg_conv_geom& g, const float* dy, const float* w, float* dx_seen,
                    const float* addend, const float* mask_src, float mask_slope, cudaStream_t st) {
    CG_REQUIRE(g.KH % g.stride == 0 && g.KW % g.stride == 0, "dgrad: kernel %dx%d not divisible by stride %d",
               g.KH, g.KW, g.stride);
    ConvKP p = make_kp(g);
    p.x = dy; p.w = w; p.y = dx_seen; p.addend = addend; p.mask_src = mask_src; p.slope = mask_slope;
    int s = g.stride;
    long Mc = (long)g.B * cdiv(p.Hin, s) * cdiv(p.Win, s);
    dim3 grid(cdiv(Mc, BM), cdiv(p.Cin, BN), p.G * s * s);
    launch_k(conv_dgrad_simt_kernel, grid, NT, 0, st, p);
    return check_launch("conv_dgrad_simt");
}

// ------------------------------------------------------------------------------------------------
// weight gradient (split-K over pixels, deterministic two-phase reduction)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) conv_wgrad_simt_kernel(ConvKP p) {
    pdl_trigger();
    pdl_wait();
    __shared__ __align__(16) float As[BK][BM + SPAD];  // [pixel][co]
    __shared__ __align__(16) float Bs[BK][BN + SPAD];  // [pixel][n]
    const int tid = threadIdx.x;
    const int g = blockIdx.z / p.splits;
    const int sp = blockIdx.z - g * p.splits;
    const int co0 = blockIdx.y * BM;
    const int n0 = blockIdx.x * BN;
    const int kk = tid >> 4, q = tid & 15;
    const int ty = tid >> 4, tx = tid & 15;
    const long mbeg = (long)sp * p.chunk;
    const long mend = min(p.Mpix, mbeg + p.chunk);

    const int co = co0 + q * 4;
    const bool vecA = (p.Cout & 3) == 0;
    const int n = n0 + q * 4;
    const bool nvalid = n < p.Ktot;
    int kh = 0, kw = 0, ci = 0;
    if (nvalid) {
        int tap = n / p.Cin;
        ci = n - tap * p.Cin;
        kh = tap / p.KW;
        kw = tap - kh * p.KW;
    }
    const float* dyb = p.y + (long)g * p.Mpix * p.Cout;  // p.y carries dy (const use)
    const float* xb = p.x + (long)g * p.xg;
    const int hw = p.Ho * p.Wo;

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.f;

    float4 ra, rb;
    auto load = [&](long mt) {
        long m = mt + kk;
        ra = make_float4(0.f, 0.f, 0.f, 0.f);
        rb = ra;
        if (m < mend) {
            const float* dp = dyb + m * p.Cout + co;
            if (vecA) {
                if (co < p.Cout) ra = ldg4(dp);
            } else {
                if (co < p.Cout) ra.x = __ldg(dp);
                if (co + 1 < p.Cout) ra.y = __ldg(dp + 1);
                if (co + 2 < p.Cout) ra.z = __ldg(dp + 2);
                if (co + 3 < p.Cout) ra.w = __ldg(dp + 3);
            }
            if (nvalid) {
                int b = (int)(m / hw);
                int r = (int)(m - (long)b * hw);
                int oh = r / p.Wo, ow = r - oh * p.Wo;
                int ih = oh * p.stride - p.pad + kh, iw = ow * p.stride - p.pad + kw;
                if (ih >= 0 && ih < p.Hin && iw >= 0 && iw < p.Win) {
                    if (p.ups) { ih >>= 1; iw >>= 1; }
                    rb = ldg4(xb + (((long)b * p.H + ih) * p.W + iw) * p.Cin + ci);
                }
            }
        }
    };
    auto store = [&]() {
        *reinterpret_cast<float4*>(&As[kk][q * 4]) = ra;
        *reinterpret_cast<float4*>(&Bs[kk][q * 4]) = rb;
    };
    if (mbeg < mend) {
        load(mbeg);
        store();
        __syncthreads();
        for (long mt = mbeg; mt < mend; mt += BK) {
            bool more = mt + BK < mend;
            if (more) load(mt + BK);
#pragma unroll
            for (int k2 = 0; k2 < BK; k2++) {
                float4 a = *reinterpret_cast<const float4*>(&As[k2][ty * 4]);
                float4 b = *reinterpret_cast<const float4*>(&Bs[k2][tx * 4]);
                float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                for (int i = 0; i < 4; i++)
#pragma unroll
                    for (int j = 0; j < 4; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
            }
            __syncthreads();
            if (more) {
                store();
                __syncthreads();
            }
        }
    }
    // out[(sp*G + g)][co][n]  (p.w carries the output pointer)
    float* out = const_cast<float*>(p.w) + ((long)sp * p.G + g) * p.Cout * p.Ktot;
    const int nn = n0 + tx * 4;
    if (nn >= p.Ktot) return;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        int c = co0 + ty * 4 + i;
        if (c >= p.Cout) continue;
        *reinterpret_cast<float4*>(out + (long)c * p.Ktot + nn) =
            make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    }
}

__global__ void reduce_splits_kernel(const float* __restrict__ part, float* __restrict__ out, long n4, int splits) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k = 0; k < splits; k++) {
        float4 v = ldg4(part + ((long)k * n4 + i) * 4);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    reinterpret_cast<float4*>(out)[i] = s;
}

static void wgrad_plan(const cg_conv_geom& g, int& splits, long& chunk) {
    ConvDims d = conv_dims(g);
    long tiles = (long)cdiv(d.Ktot, BN) * cdiv(g.Cout, BM) * g.G;
    long want = cdiv(592, tiles);
    long maxs = cdiv(d.Mpix, 256);
    splits = (int)(want < maxs ? want : maxs);
    if (splits < 1) splits = 1;
    if (splits > 64) splits = 64;
    chunk = (cdiv(d.Mpix, splits) + BK - 1) / BK * BK;
    splits = cdiv(d.Mpix, chunk);
}

size_t simt_wgrad_ws(const cg_conv_geom& g) {
    int splits; long chunk;
    wgrad_plan(g, splits, chunk);
    if (splits == 1) return 0;
    ConvDims d = conv_dims(g);
    return (size_t)splits * g.G * g.Cout * d.Ktot * sizeof(float);
}

int simt_conv_wgrad(const cg_conv_geom& g, const float* x, const float* dy, float* dw, void* ws,
                    size_t ws_bytes, cudaStream_t st) {
    ConvKP p = make_kp(g);
    wgrad_plan(g, p.splits, p.chunk);
    size_t need = simt_wgrad_ws(g);
    if (need > ws_bytes) {
        set_error("conv_wgrad: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    float* out = p.splits == 1 ? dw : reinterpret_cast<float*>(ws);
    p.x = x; p.y = const_cast<float*>(dy); p.w = out;
    dim3 grid(cdiv(p.Ktot, BN), cdiv(p.Cout, BM), p.G * p.splits);
    launch_k(conv_wgrad_simt_kernel, grid, NT, 0, st, p);
    int rc = check_launch("conv_wgrad_simt");
    if (rc) return rc;
    if (p.splits > 1) {
        long n4 = (long)p.G * p.Cout * p.Ktot / 4;
        launch_k(reduce_splits_kernel, cdiv(n4, 256), 256, 0, st, out, dw, n4, p.splits);
        rc = check_launch("reduce_splits");
    }
    return rc;
}

// ------------------------------------------------------------------------------------------------
// column sums (bias gradient): db[g][c] = sum_rows dy[g][row][c]
// ------------------------------------------------------------------------------------------------
// rows per partial sum: >= 128 and at most 256 partials per group, so the 64x64x256 maps launch 1024 blocks instead of 128
static inline int cs_rows(long rows) {
    long r = (rows + 255) / 256;
    r = (r + 63) / 64 * 64;
    return (int)(r < 128 ? 128 : r);
}
__global__ void __launch_bounds__(256) colsum_partial_kernel(const float* __restrict__ dy, float* __restrict__ part,
                                                             long rows, int C, int nchunks, int CS_ROWS) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sm[256];
    const int g = blockIdx.y, chunk = blockIdx.x;
    const int cpp = C < 256 ? C : 256;
    const int rl_n = 256 / cpp;
    const int tid = threadIdx.x;
    const int c_in = tid % cpp, rl = tid / cpp;
    const long r0 = (long)chunk * CS_ROWS, r1 = min(rows, r0 + CS_ROWS);
    const float* base = dy + (long)g * rows * C;
    for (int cb = 0; cb < C; cb += cpp) {
        int c = cb + c_in;
        float s = 0.f;
        if (rl < rl_n && c < C)
            for (long r = r0 + rl; r < r1; r += rl_n) s += __ldg(base + r * C + c);
        sm[tid] = s;
        __syncthreads();
        if (rl == 0 && c < C) {
            float t = 0.f;
            for (int k = 0; k < rl_n; k++) t += sm[k * cpp + c_in];
            part[((long)chunk * gridDim.y + g) * C + c] = t;
        }
        __syncthreads();
    }
}
__global__ void colsum_final_kernel(const float* __restrict__ part, float* __restrict__ out, int GC, int nchunks) {
    pdl_trigger();
    pdl_wait();
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= GC) return;
    float s = 0.f;
    for (int k = 0; k < nchunks; k++) s += part[(long)k * GC + i];
    out[i] = s;
}
// float4-vectorised variant for C % 4 == 0, C/4 dividing 256: lanes = C/4 threads across channels, 256/lanes row lanes
__global__ void __launch_bounds__(256) colsum_partial_v4_kernel(const float* __restrict__ dy, float* __restrict__ part, long rows, int C,
                                                                int CS_ROWS) {
    pdl_trigger();
    pdl_wait();
    __shared__ float4 sm[256];
    const int g = blockIdx.y, chunk = blockIdx.x;
    const int lanes = C >> 2, rowl = 256 / lanes;
    const int lane = threadIdx.x % lanes, rl = threadIdx.x / lanes;
    const long r0 = (long)chunk * CS_ROWS, r1 = min(rows, r0 + CS_ROWS);
    const float* base = dy + (long)g * rows * C + lane * 4;
    float4 s0 = make_float4(0.f, 0.f, 0.f, 0.f), s1 = s0;
    for (long r = r0 + rl; r < r1; r += 4 * rowl) {  // four independent 16-byte loads in flight per thread
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const long rr = r + (long)u * rowl;
            v[u] = rr < r1 ? __ldg(reinterpret_cast<const float4*>(base + rr * C)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        s0.x += v[0].x + v[2].x; s0.y += v[0].y + v[2].y; s0.z += v[0].z + v[2].z; s0.w += v[0].w + v[2].w;
        s1.x += v[1].x + v[3].x; s1.y += v[1].y + v[3].y; s1.z += v[1].z + v[3].z; s1.w += v[1].w + v[3].w;
    }
    s0.x += s1.x; s0.y += s1.y; s0.z += s1.z; s0.w += s1.w;
    sm[threadIdx.x] = s0;
    __syncthreads();
    if (rl == 0) {
        for (int k = 1; k < rowl; k++) {
            float4 a = sm[k * lanes + lane];
            s0.x += a.x; s0.y += a.y; s0.z += a.z; s0.w += a.w;
        }
        *reinterpret_cast<float4*>(part + ((long)chunk * gridDim.y + g) * C + lane * 4) = s0;
    }
}
size_t colsum_ws(int G, long rows, int C) { return (size_t)cdiv(rows, cs_rows(rows)) * G * C * sizeof(float); }
int colsum(const float* dy, float* db, int G, long rows, int C, void* ws, size_t ws_bytes, cudaStream_t st) {
    size_t need = colsum_ws(G, rows, C);
    if (need > ws_bytes) {
        set_error("colsum: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    const int csr = cs_rows(rows);
    int nchunks = cdiv(rows, csr);
    if (C % 4 == 0 && C / 4 <= 256 && 256 % (C / 4) == 0)
        launch_k(colsum_partial_v4_kernel, dim3(nchunks, G), 256, 0, st, dy, (float*)ws, rows, C, csr);
    else
        launch_k(colsum_partial_kernel, dim3(nchunks, G), 256, 0, st, dy, (float*)ws, rows, C, nchunks, csr);
    int rc = check_launch("colsum_partial");
    if (rc) return rc;
    launch_k(colsum_final_kernel, cdiv((long)G * C, 256), 256, 0, st, (const float*)ws, db, G * C, nchunks);
    return check_launch("colsum_final");
}

// ------------------------------------------------------------------------------------------------
// 2x2 fan-in sum of the nearest-upsample (backward of nn.Upsample(scale_factor=2), networks.py:385)
// dx[n][h][w][c] = (sum_{i,j<2} d_up[n][2h+i][2w+j][c] [+ addend]) * act'(mask_src)
// ------------------------------------------------------------------------------------------------
__global__ void pool2x2_sum_kernel(const float* __restrict__ d_up, float* __restrict__ dx, const float* __restrict__ addend,
                                   const float* __restrict__ mask_src, float slope, long total4, int H, int W, int C4) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total4) return;
    int c = (int)(i % C4);
    long pix = i / C4;
    int w = (int)(pix % W);
    long t = pix / W;
    int h = (int)(t % H);
    long n = t / H;
    const float4* src = reinterpret_cast<const float4*>(d_up);
    long W2 = 2L * W;
    long base = ((n * 2 * H + 2 * h) * W2 + 2 * w) * C4 + c;
    float4 a = __ldg(src + base), b = __ldg(src + base + C4), cc = __ldg(src + base + W2 * C4),
           d = __ldg(src + base + W2 * C4 + C4);
    float4 v = make_float4(a.x + b.x + cc.x + d.x, a.y + b.y + cc.y + d.y, a.z + b.z + cc.z + d.z, a.w + b.w + cc.w + d.w);
    if (addend) {
        float4 e = __ldg(reinterpret_cast<const float4*>(addend) + i);
        v.x += e.x; v.y += e.y; v.z += e.z; v.w += e.w;
    }
    if (mask_src) {
        float4 e = __ldg(reinterpret_cast<const float4*>(mask_src) + i);
        v.x *= e.x > 0.f ? 1.f : slope; v.y *= e.y > 0.f ? 1.f : slope;
        v.z *= e.z > 0.f ? 1.f : slope; v.w *= e.w > 0.f ? 1.f : slope;
    }
    reinterpret_cast<float4*>(dx)[i] = v;
}
int pool2x2_sum(const float* d_up, float* dx, const float* addend, const float* mask_src, float mask_slope,
                long N, int H, int W, int C, cudaStream_t st) {
    long total4 = N * H * W * (C / 4);
    launch_k(pool2x2_sum_kernel, cdiv(total4, 256), 256, 0, st, d_up, dx, addend, mask_src, mask_slope, total4, H, W, C / 4);
    return check_launch("pool2x2_sum");
}

}  // namespace cg
