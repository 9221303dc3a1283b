// Instance norm / AdaIN / layer norm statistics, apply(+activation,+residual,+x2 upsample) and backward.
//
// Reference call sites replaced: nn.InstanceNorm2d (networks.py:483,518), AdaptiveInstanceNorm2d via
// F.batch_norm on (1, B*C, H, W) (networks.py:640-653), LayerNorm (networks.py:659-686, the discriminators'
// norm: ln), the in-place ReLU / LeakyReLU(0.2) (networks.py:493-495,520), the residual add (networks.py:460)
// and nn.Upsample(scale_factor=2) (networks.py:385), plus their autograd.
//
// All tensors channels-last [G][B][HW][C]; HBM-bound: every kernel streams float4 along C.
#include "common.cuh"

namespace cg {

constexpr int ST_ROWS = 128;  // pixels per block (and per partial sum): 1024+ blocks on the 64x64x256 maps, one resident wave
constexpr int ST_U = 4;       // rows in flight per thread: independent 16-byte loads issued before their first use

// lanes = C/4 threads span the channel axis, 256/lanes threads stride the pixel axis.
struct LaneMap {
    int lanes, rowl, lane, rl;
    __device__ LaneMap(int C) {
        lanes = C >> 2;
        rowl = 256 / lanes;
        lane = threadIdx.x % lanes;
        rl = threadIdx.x / lanes;
    }
};

__device__ __forceinline__ float4 f4ld(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// ---- statistics --------------------------------------------------------------------------------
// part[chunk][gb][C][2] = (sum, sum of squares) of a pixel chunk
__global__ void __launch_bounds__(256) in_stats_partial_kernel(const float* __restrict__ y, float* __restrict__ part,
                                                               int HW, int C) {
    pdl_trigger();
    pdl_wait();
    __shared__ float4 sm[2][256];
    const int gb = blockIdx.y, chunk = blockIdx.x;
    LaneMap lm(C);
    const int r0 = chunk * ST_ROWS, r1 = min(HW, r0 + ST_ROWS);
    const float* base = y + ((long)gb * HW) * C + lm.lane * 4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = s;
    if (lm.rl < lm.rowl)
        for (int r = r0 + lm.rl; r < r1; r += ST_U * lm.rowl) {
            float4 v[ST_U];
#pragma unroll
            for (int u = 0; u < ST_U; u++) {
                const int rr = r + u * lm.rowl;
                v[u] = rr < r1 ? f4ld(base + (long)rr * C) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < ST_U; u++) {
                s.x += v[u].x; s.y += v[u].y; s.z += v[u].z; s.w += v[u].w;
                q.x += v[u].x * v[u].x; q.y += v[u].y * v[u].y; q.z += v[u].z * v[u].z; q.w += v[u].w * v[u].w;
            }
        }
    sm[0][threadIdx.x] = s;
    sm[1][threadIdx.x] = q;
    __syncthreads();
    if (lm.rl == 0) {
        for (int k = 1; k < lm.rowl; k++) {
            float4 a = sm[0][k * lm.lanes + lm.lane], b = sm[1][k * lm.lanes + lm.lane];
            s.x += a.x; s.y += a.y; s.z += a.z; s.w += a.w;
            q.x += b.x; q.y += b.y; q.z += b.z; q.w += b.w;
        }
        float* o = part + (((long)chunk * gridDim.y + gb) * C + lm.lane * 4) * 2;
        o[0] = s.x; o[1] = q.x; o[2] = s.y; o[3] = q.y; o[4] = s.z; o[5] = q.z; o[6] = s.w; o[7] = q.w;
    }
}
// 32 items x 8 chunk slices per block: the chunk loop of one (gb, c) item is split eight ways and folded in shared memory
// (fp64), so the 256x256 maps (512 chunks, only 2048 items) do not serialise 512 dependent loads per thread.
constexpr int FIN_ITEMS = 32, FIN_SLICES = 8;
__device__ __forceinline__ bool final_sums(const float* __restrict__ part, long GBC, int nchunks, long i, double& s, double& q) {
    __shared__ double sm[2][FIN_SLICES][FIN_ITEMS];
    s = 0.0; q = 0.0;
    if (i < GBC)
        for (int k = threadIdx.y; k < nchunks; k += FIN_SLICES) {
            float2 v = __ldg(reinterpret_cast<const float2*>(part + ((long)k * GBC + i) * 2));
            s += (double)v.x;
            q += (double)v.y;
        }
    sm[0][threadIdx.y][threadIdx.x] = s;
    sm[1][threadIdx.y][threadIdx.x] = q;
    __syncthreads();
    if (threadIdx.y != 0 || i >= GBC) return false;
    for (int k = 1; k < FIN_SLICES; k++) {
        s += sm[0][k][threadIdx.x];
        q += sm[1][k][threadIdx.x];
    }
    return true;
}
__global__ void __launch_bounds__(FIN_ITEMS * FIN_SLICES) in_stats_final_kernel(const float* __restrict__ part, float* __restrict__ mean,
                                                                                 float* __restrict__ rstd, long GBC, int nchunks, int HW,
                                                                                 float eps) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * FIN_ITEMS + threadIdx.x;
    double s, q;
    if (!final_sums(part, GBC, nchunks, i, s, q)) return;
    double m = s / HW;
    double var = q / HW - m * m;
    if (var < 0.0) var = 0.0;
    mean[i] = (float)m;
    rstd[i] = (float)(1.0 / sqrt(var + (double)eps));
}

// ---- forward apply -----------------------------------------------------------------------------
// Layer norm (the kernels' LN instances): mean = ln mean[gb], rstd = 1 / (std[gb] + eps) with the per-sample statistics of
// cg_ln_stats in mean / rstd's place (rstd holds the std), gamma / beta per member and channel ln_gamma[g][C] / ln_beta[g][C].
struct NormP {
    const float* y; const float* mean; const float* rstd; const float* adain; const float* res;
    const float* dz; float* z; float* dy; float* part; float* d_adain;
    const float* ln_gamma; const float* ln_beta;
    int P, off, B, H, W, C, act, ups;
    float ln_eps;
};

constexpr float LRELU_SLOPE = 0.2f;  // nn.LeakyReLU(0.2), fixed by Conv2dBlock (networks.py:493)

// Kernel instances: instance norm / AdaIN with ReLU or none (the generators), with LeakyReLU as well (the discriminators' in),
// and layer norm.  Separate instances keep the generators' kernels at their register counts.
enum NormMode { NM_IN = 0, NM_IN_LRELU = 1, NM_LN = 2 };

// the normalisation's mean and 1/std of channels c..c+3 of sample gb
template <int M>
__device__ __forceinline__ void stats_for(const NormP& p, int gb, int c, float4& mu, float4& rs) {
    if (M == NM_LN) {
        const float m = __ldg(p.mean + gb), r = 1.f / (__ldg(p.rstd + gb) + p.ln_eps);
        mu = make_float4(m, m, m, m);
        rs = make_float4(r, r, r, r);
        return;
    }
    mu = f4ld(p.mean + (long)gb * p.C + c);
    rs = f4ld(p.rstd + (long)gb * p.C + c);
}

__device__ __forceinline__ float4 ln_gamma_for(const NormP& p, int gb, int c) {
    return f4ld(p.ln_gamma + (long)(gb / p.B) * p.C + c);
}

// g1 = dz * act'(pre): ReLU passes nothing at pre <= 0, LeakyReLU passes slope (torch's gradients at 0)
#define CG_ACT_GRAD(g1, v, a, b)                                                                             \
    if (p.act == CG_ACT_RELU) {                                                                             \
        if (fmaf(v.x, a.x, b.x) <= 0.f) g1.x = 0.f;                                                         \
        if (fmaf(v.y, a.y, b.y) <= 0.f) g1.y = 0.f;                                                         \
        if (fmaf(v.z, a.z, b.z) <= 0.f) g1.z = 0.f;                                                         \
        if (fmaf(v.w, a.w, b.w) <= 0.f) g1.w = 0.f;                                                         \
    } else if (M != NM_IN && p.act == CG_ACT_LRELU) {                                                       \
        if (fmaf(v.x, a.x, b.x) <= 0.f) g1.x *= LRELU_SLOPE;                                                \
        if (fmaf(v.y, a.y, b.y) <= 0.f) g1.y *= LRELU_SLOPE;                                                \
        if (fmaf(v.z, a.z, b.z) <= 0.f) g1.z *= LRELU_SLOPE;                                                \
        if (fmaf(v.w, a.w, b.w) <= 0.f) g1.w *= LRELU_SLOPE;                                                \
    }

template <int M>
__device__ __forceinline__ void affine_for(const NormP& p, int gb, int c, float4& a, float4& b) {
    float4 mu, rs;
    stats_for<M>(p, gb, c, mu, rs);
    float4 ga = make_float4(1.f, 1.f, 1.f, 1.f), be = make_float4(0.f, 0.f, 0.f, 0.f);
    if (M == NM_LN) {
        ga = ln_gamma_for(p, gb, c);
        be = f4ld(p.ln_beta + (long)(gb / p.B) * p.C + c);
    } else if (p.adain) {
        const float* ap = p.adain + (long)gb * p.P + p.off;
        be = f4ld(ap + c);
        ga = f4ld(ap + p.C + c);
    }
    a = make_float4(ga.x * rs.x, ga.y * rs.y, ga.z * rs.z, ga.w * rs.w);
    b = make_float4(be.x - mu.x * a.x, be.y - mu.y * a.y, be.z - mu.z * a.z, be.w - mu.w * a.w);
}

// three blocks per SM, as these streaming kernels reach at their natural register count
template <int M>
__global__ void __launch_bounds__(256, 3) norm_act_fwd_kernel(NormP p) {
    pdl_trigger();
    pdl_wait();
    const int gb = blockIdx.y;
    const int HW = p.H * p.W;
    LaneMap lm(p.C);
    if (lm.rl >= lm.rowl) return;
    const int c = lm.lane * 4;
    float4 a, b;
    affine_for<M>(p, gb, c, a, b);
    const int r0 = blockIdx.x * ST_ROWS, r1 = min(HW, r0 + ST_ROWS);
    const float* yb = p.y + (long)gb * HW * p.C + c;
    const float* rb = p.res ? p.res + (long)gb * HW * p.C + c : nullptr;
    for (int r = r0 + lm.rl; r < r1; r += ST_U * lm.rowl) {
        float4 v[ST_U], e[ST_U];
#pragma unroll
        for (int u = 0; u < ST_U; u++) {
            const int rr = r + u * lm.rowl;
            if (rr < r1) {
                v[u] = f4ld(yb + (long)rr * p.C);
                if (rb) e[u] = f4ld(rb + (long)rr * p.C);
            }
        }
#pragma unroll
        for (int u = 0; u < ST_U; u++) {
            const int rr = r + u * lm.rowl;
            if (rr >= r1) break;
            float4 o;
            o.x = fmaf(v[u].x, a.x, b.x); o.y = fmaf(v[u].y, a.y, b.y); o.z = fmaf(v[u].z, a.z, b.z); o.w = fmaf(v[u].w, a.w, b.w);
            if (p.act == CG_ACT_RELU) {
                o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f);
            } else if (M != NM_IN && p.act == CG_ACT_LRELU) {
                o.x = o.x > 0.f ? o.x : o.x * LRELU_SLOPE; o.y = o.y > 0.f ? o.y : o.y * LRELU_SLOPE;
                o.z = o.z > 0.f ? o.z : o.z * LRELU_SLOPE; o.w = o.w > 0.f ? o.w : o.w * LRELU_SLOPE;
            }
            if (rb) {
                o.x += e[u].x; o.y += e[u].y; o.z += e[u].z; o.w += e[u].w;
            }
            if (!p.ups) {
                *reinterpret_cast<float4*>(p.z + ((long)gb * HW + rr) * p.C + c) = o;
            } else {
                int h = rr / p.W, w = rr - h * p.W;
                long W2 = 2L * p.W;
                float* zp = p.z + (((long)gb * 2 * p.H + 2 * h) * W2 + 2 * w) * p.C + c;
                *reinterpret_cast<float4*>(zp) = o;
                *reinterpret_cast<float4*>(zp + p.C) = o;
                *reinterpret_cast<float4*>(zp + W2 * p.C) = o;
                *reinterpret_cast<float4*>(zp + W2 * p.C + p.C) = o;
            }
        }
    }
}

// ---- backward ----------------------------------------------------------------------------------
__device__ __forceinline__ float4 load_dz(const NormP& p, int gb, int r, int c) {
    if (!p.ups) return f4ld(p.dz + ((long)gb * p.H * p.W + r) * p.C + c);
    int h = r / p.W, w = r - h * p.W;
    long W2 = 2L * p.W;
    const float* zp = p.dz + (((long)gb * 2 * p.H + 2 * h) * W2 + 2 * w) * p.C + c;
    float4 a = f4ld(zp), b = f4ld(zp + p.C), cc = f4ld(zp + W2 * p.C), d = f4ld(zp + W2 * p.C + p.C);
    return make_float4(a.x + b.x + cc.x + d.x, a.y + b.y + cc.y + d.y, a.z + b.z + cc.z + d.z, a.w + b.w + cc.w + d.w);
}

// phase 1: part[chunk][gb][C][2] = (sum g1, sum g1*xhat), g1 = dz * act'(pre)
template <int M>
__global__ void __launch_bounds__(256) norm_bwd_partial_kernel(NormP p) {
    pdl_trigger();
    pdl_wait();
    __shared__ float4 sm[2][256];
    const int gb = blockIdx.y;
    const int HW = p.H * p.W;
    LaneMap lm(p.C);
    const int c = lm.lane * 4;
    float4 a, b, mu, rs;
    affine_for<M>(p, gb, c, a, b);
    stats_for<M>(p, gb, c, mu, rs);
    const int r0 = blockIdx.x * ST_ROWS, r1 = min(HW, r0 + ST_ROWS);
    const float* yb = p.y + (long)gb * HW * p.C + c;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f), q = s;
    if (lm.rl < lm.rowl)
        for (int r = r0 + lm.rl; r < r1; r += ST_U * lm.rowl) {
            float4 vv[ST_U], gg[ST_U];
#pragma unroll
            for (int u = 0; u < ST_U; u++) {
                const int rr = r + u * lm.rowl;
                if (rr < r1) {
                    vv[u] = f4ld(yb + (long)rr * p.C);
                    gg[u] = load_dz(p, gb, rr, c);
                } else {
                    vv[u] = mu;
                    gg[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
#pragma unroll
            for (int u = 0; u < ST_U; u++) {
                float4 v = vv[u], g1 = gg[u];
                CG_ACT_GRAD(g1, v, a, b)
                s.x += g1.x; s.y += g1.y; s.z += g1.z; s.w += g1.w;
                q.x += g1.x * (v.x - mu.x) * rs.x; q.y += g1.y * (v.y - mu.y) * rs.y;
                q.z += g1.z * (v.z - mu.z) * rs.z; q.w += g1.w * (v.w - mu.w) * rs.w;
            }
        }
    sm[0][threadIdx.x] = s;
    sm[1][threadIdx.x] = q;
    __syncthreads();
    if (lm.rl == 0) {
        for (int k = 1; k < lm.rowl; k++) {
            float4 aa = sm[0][k * lm.lanes + lm.lane], bb = sm[1][k * lm.lanes + lm.lane];
            s.x += aa.x; s.y += aa.y; s.z += aa.z; s.w += aa.w;
            q.x += bb.x; q.y += bb.y; q.z += bb.z; q.w += bb.w;
        }
        float* o = p.part + (((long)blockIdx.x * gridDim.y + gb) * p.C + c) * 2;
        o[0] = s.x; o[1] = q.x; o[2] = s.y; o[3] = q.y; o[4] = s.z; o[5] = q.z; o[6] = s.w; o[7] = q.w;
    }
}
// sums[gb][C][2] (fp32) = chunk totals; also scatters d_beta / d_gamma into d_adain
__global__ void __launch_bounds__(FIN_ITEMS * FIN_SLICES) norm_bwd_final_kernel(const float* __restrict__ part, float* __restrict__ sums,
                                                                                 float* __restrict__ d_adain, int GB, int C, int P, int off,
                                                                                 int nchunks) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * FIN_ITEMS + threadIdx.x;
    long GBC = (long)GB * C;
    double s, q;
    if (!final_sums(part, GBC, nchunks, i, s, q)) return;
    sums[i * 2] = (float)s;
    sums[i * 2 + 1] = (float)q;
    if (d_adain) {
        int gb = (int)(i / C), c = (int)(i - (long)gb * C);
        d_adain[(long)gb * P + off + c] = (float)s;       // d beta  ("mean" columns)
        d_adain[(long)gb * P + off + C + c] = (float)q;   // d gamma ("std" columns)
    }
}
// phase 2: dy = gamma*rstd * (g1 - mean(g1) - xhat*mean(g1*xhat));
// layer norm: dy = rstd * (gamma*g1 - k1 - (y - mean) * k2) with the per-sample k1, k2 of ln_bwd_final_kernel in sums[gb][2]
template <int M>
__global__ void __launch_bounds__(256, 3) norm_bwd_apply_kernel(NormP p, const float* __restrict__ sums) {
    pdl_trigger();
    pdl_wait();
    const int gb = blockIdx.y;
    const int HW = p.H * p.W;
    LaneMap lm(p.C);
    if (lm.rl >= lm.rowl) return;
    const int c = lm.lane * 4;
    float4 a, b, mu, rs;
    affine_for<M>(p, gb, c, a, b);
    stats_for<M>(p, gb, c, mu, rs);
    float m1[4], m2[4];
    float4 ga = make_float4(1.f, 1.f, 1.f, 1.f);
    if (M == NM_LN) {
        ga = ln_gamma_for(p, gb, c);
        m1[0] = m1[1] = m1[2] = m1[3] = sums[gb * 2];
        m2[0] = m2[1] = m2[2] = m2[3] = sums[gb * 2 + 1];
    } else {
        const float* sp = sums + ((long)gb * p.C + c) * 2;
        const float inv = 1.f / (float)HW;
        m1[0] = sp[0] * inv; m1[1] = sp[2] * inv; m1[2] = sp[4] * inv; m1[3] = sp[6] * inv;
        m2[0] = sp[1] * inv; m2[1] = sp[3] * inv; m2[2] = sp[5] * inv; m2[3] = sp[7] * inv;
    }
    const int r0 = blockIdx.x * ST_ROWS, r1 = min(HW, r0 + ST_ROWS);
    const float* yb = p.y + (long)gb * HW * p.C + c;
    for (int r = r0 + lm.rl; r < r1; r += ST_U * lm.rowl) {
        float4 vv[ST_U], gg[ST_U];
#pragma unroll
        for (int u = 0; u < ST_U; u++) {
            const int rr = r + u * lm.rowl;
            if (rr < r1) {
                vv[u] = f4ld(yb + (long)rr * p.C);
                gg[u] = load_dz(p, gb, rr, c);
            }
        }
#pragma unroll
        for (int u = 0; u < ST_U; u++) {
            const int rr = r + u * lm.rowl;
            if (rr >= r1) break;
            float4 v = vv[u], g1 = gg[u];
            CG_ACT_GRAD(g1, v, a, b)
            float4 o;
            if (M == NM_LN) {
                o.x = rs.x * (ga.x * g1.x - m1[0] - (v.x - mu.x) * m2[0]);
                o.y = rs.y * (ga.y * g1.y - m1[1] - (v.y - mu.y) * m2[1]);
                o.z = rs.z * (ga.z * g1.z - m1[2] - (v.z - mu.z) * m2[2]);
                o.w = rs.w * (ga.w * g1.w - m1[3] - (v.w - mu.w) * m2[3]);
            } else {
                o.x = a.x * (g1.x - m1[0] - (v.x - mu.x) * rs.x * m2[0]);
                o.y = a.y * (g1.y - m1[1] - (v.y - mu.y) * rs.y * m2[1]);
                o.z = a.z * (g1.z - m1[2] - (v.z - mu.z) * rs.z * m2[2]);
                o.w = a.w * (g1.w - m1[3] - (v.w - mu.w) * rs.w * m2[3]);
            }
            *reinterpret_cast<float4*>(p.dy + ((long)gb * HW + rr) * p.C + c) = o;
        }
    }
}

// ---- layer norm (LayerNorm networks.py:659-686): per-sample statistics over C x H x W ------------------------------
// Both reductions fold a sample's (chunk, channel) partials in a fixed order: a strided fp64 sum per thread, then a fixed
// shared-memory tree, so the results do not depend on scheduling.
constexpr int LN_THREADS = 256;
__device__ __forceinline__ void block_sum2(double& s, double& q) {
    __shared__ double sm[2][LN_THREADS];
    sm[0][threadIdx.x] = s;
    sm[1][threadIdx.x] = q;
    __syncthreads();
    for (int k = LN_THREADS / 2; k > 0; k >>= 1) {
        if ((int)threadIdx.x < k) {
            sm[0][threadIdx.x] += sm[0][threadIdx.x + k];
            sm[1][threadIdx.x] += sm[1][threadIdx.x + k];
        }
        __syncthreads();
    }
    s = sm[0][0];
    q = sm[1][0];
}

// mean[gb] and the unbiased std[gb] (torch.std) from part[chunk][gb][C][2] = (sum, sum of squares) of in_stats_partial_kernel
__global__ void __launch_bounds__(LN_THREADS) ln_stats_final_kernel(const float* __restrict__ part, float* __restrict__ mean,
                                                                     float* __restrict__ std, int GB, int C, int nchunks, long N) {
    pdl_trigger();
    pdl_wait();
    const int gb = blockIdx.x;
    double s = 0.0, q = 0.0;
    for (int k = threadIdx.x; k < nchunks * C; k += LN_THREADS) {
        const int chunk = k / C, c = k - chunk * C;
        float2 v = __ldg(reinterpret_cast<const float2*>(part + (((long)chunk * GB + gb) * C + c) * 2));
        s += (double)v.x;
        q += (double)v.y;
    }
    block_sum2(s, q);
    if (threadIdx.x != 0) return;
    const double m = s / (double)N;
    double var = (q - s * m) / (double)(N - 1);
    if (var < 0.0) var = 0.0;
    mean[gb] = (float)m;
    std[gb] = (float)sqrt(var);
}

// From part[chunk][gb][C][2] = (sum g1, sum g1*xhat) of norm_bwd_partial_kernel: cs[gb][C][2] = the chunk totals (what dgamma /
// dbeta sum over the batch) and sums[gb] = (k1, k2) of the apply pass,
//   k1 = sum(gamma*g1) / N,  k2 = sum(gamma*g1*xhat) / ((N-1) * std)
// (the autograd of (y - mean) / (std + eps) with the unbiased std: d std / d y = (y - mean) / ((N-1) * std); 0 at std 0).
__global__ void __launch_bounds__(LN_THREADS) ln_bwd_final_kernel(const float* __restrict__ part, const float* __restrict__ gamma,
                                                                   const float* __restrict__ std, float* __restrict__ cs,
                                                                   float* __restrict__ sums, int GB, int B, int C, int nchunks, long N) {
    pdl_trigger();
    pdl_wait();
    const int gb = blockIdx.x;
    double a = 0.0, q = 0.0;
    for (int c = threadIdx.x; c < C; c += LN_THREADS) {
        double s1 = 0.0, s2 = 0.0;
        for (int k = 0; k < nchunks; k++) {
            float2 v = __ldg(reinterpret_cast<const float2*>(part + (((long)k * GB + gb) * C + c) * 2));
            s1 += (double)v.x;
            s2 += (double)v.y;
        }
        cs[((long)gb * C + c) * 2] = (float)s1;
        cs[((long)gb * C + c) * 2 + 1] = (float)s2;
        const double ga = (double)__ldg(gamma + (long)(gb / B) * C + c);
        a += ga * s1;
        q += ga * s2;
    }
    block_sum2(a, q);
    if (threadIdx.x != 0) return;
    const double sd = (double)std[gb];
    sums[gb * 2] = (float)(a / (double)N);
    sums[gb * 2 + 1] = sd > 0.0 ? (float)(q / ((double)(N - 1) * sd)) : 0.f;
}

// dbeta[g][c] = sum over the member's samples of sum g1, dgamma[g][c] = of sum g1*xhat (overwritten, in sample order)
__global__ void __launch_bounds__(256) ln_param_grad_kernel(const float* __restrict__ cs, float* __restrict__ dgamma,
                                                            float* __restrict__ dbeta, int G, int B, int C) {
    pdl_trigger();
    pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)G * C) return;
    const int g = (int)(i / C), c = (int)(i - (long)g * C);
    double s1 = 0.0, s2 = 0.0;
    for (int b = 0; b < B; b++) {
        const float* v = cs + (((long)g * B + b) * C + c) * 2;
        s1 += (double)v[0];
        s2 += (double)v[1];
    }
    dbeta[i] = (float)s1;
    dgamma[i] = (float)s2;
}

int in_stats_finalize(const float* part, float* mean, float* rstd, long GBC, int nchunks, int HW, float eps, cudaStream_t st) {
    launch_k(in_stats_final_kernel, cdiv(GBC, FIN_ITEMS), dim3(FIN_ITEMS, FIN_SLICES), 0, st, part, mean, rstd, GBC, nchunks, HW, eps);
    return check_launch("in_stats_final");
}

static int check_c(int C) {
    CG_REQUIRE(C % 4 == 0 && C / 4 <= 256 && 256 % (C / 4) == 0, "norm: unsupported channel count %d", C);
    return CG_OK;
}

}  // namespace cg

using namespace cg;

extern "C" int cg_in_stats(const float* y, float* mean, float* rstd, int G, int B, int HW, int C, float eps,
                           void* ws, size_t ws_bytes, void* stream) {
    if (int rc = check_c(C)) return rc;
    int nchunks = cdiv(HW, ST_ROWS);
    size_t need = (size_t)nchunks * G * B * C * 2 * sizeof(float);
    if (need > ws_bytes) {
        set_error("in_stats: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    launch_k(in_stats_partial_kernel, dim3(nchunks, G * B), 256, 0, st, y, (float*)ws, HW, C);
    if (int rc = check_launch("in_stats_partial")) return rc;
    long GBC = (long)G * B * C;
    launch_k(in_stats_final_kernel, cdiv(GBC, FIN_ITEMS), dim3(FIN_ITEMS, FIN_SLICES), 0, st, (const float*)ws, mean, rstd, GBC, nchunks, HW, eps);
    return check_launch("in_stats_final");
}

extern "C" int cg_norm_act_fwd(const float* y, const float* mean, const float* rstd, const float* adain, int P,
                               int off, const float* res, float* z, int G, int B, int H, int W, int C, int act,
                               int ups, void* stream) {
    if (int rc = check_c(C)) return rc;
    CG_REQUIRE(act == CG_ACT_NONE || act == CG_ACT_RELU || act == CG_ACT_LRELU, "norm_act_fwd: activation %d unsupported", act);
    NormP p{};
    p.y = y; p.mean = mean; p.rstd = rstd; p.adain = adain; p.res = res; p.z = z;
    p.P = P; p.off = off; p.B = B; p.H = H; p.W = W; p.C = C; p.act = act; p.ups = ups;
    dim3 grid(cdiv((long)H * W, ST_ROWS), G * B);
    if (act == CG_ACT_LRELU)
        launch_k(norm_act_fwd_kernel<NM_IN_LRELU>, grid, 256, 0, (cudaStream_t)stream, p);
    else
        launch_k(norm_act_fwd_kernel<NM_IN>, grid, 256, 0, (cudaStream_t)stream, p);
    return check_launch("norm_act_fwd");
}

extern "C" int cg_norm_act_bwd(const float* dz, const float* y, const float* mean, const float* rstd,
                               const float* adain, int P, int off, float* dy, float* d_adain, int G, int B,
                               int H, int W, int C, int act, int ups, void* ws, size_t ws_bytes, void* stream) {
    if (int rc = check_c(C)) return rc;
    CG_REQUIRE(act == CG_ACT_NONE || act == CG_ACT_RELU || act == CG_ACT_LRELU, "norm_act_bwd: activation %d unsupported", act);
    int nchunks = cdiv((long)H * W, ST_ROWS);
    long GBC = (long)G * B * C;
    size_t need = ((size_t)nchunks + 1) * GBC * 2 * sizeof(float);
    if (need > ws_bytes) {
        set_error("norm_act_bwd: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    NormP p{};
    p.dz = dz; p.y = y; p.mean = mean; p.rstd = rstd; p.adain = adain; p.dy = dy; p.d_adain = d_adain;
    p.P = P; p.off = off; p.B = B; p.H = H; p.W = W; p.C = C; p.act = act; p.ups = ups;
    p.part = (float*)ws;
    float* sums = (float*)ws + (size_t)nchunks * GBC * 2;
    dim3 grid(nchunks, G * B);
    const bool lrelu = act == CG_ACT_LRELU;
    if (lrelu)
        launch_k(norm_bwd_partial_kernel<NM_IN_LRELU>, grid, 256, 0, st, p);
    else
        launch_k(norm_bwd_partial_kernel<NM_IN>, grid, 256, 0, st, p);
    if (int rc = check_launch("norm_bwd_partial")) return rc;
    launch_k(norm_bwd_final_kernel, cdiv(GBC, FIN_ITEMS), dim3(FIN_ITEMS, FIN_SLICES), 0, st, p.part, sums, adain ? d_adain : nullptr, G * B, C, P, off,
                                                                                       nchunks);
    if (int rc = check_launch("norm_bwd_final")) return rc;
    if (lrelu)
        launch_k(norm_bwd_apply_kernel<NM_IN_LRELU>, grid, 256, 0, st, p, (const float*)sums);
    else
        launch_k(norm_bwd_apply_kernel<NM_IN>, grid, 256, 0, st, p, (const float*)sums);
    return check_launch("norm_bwd_apply");
}

extern "C" size_t cg_ln_workspace_bytes(int G, int B, int HW, int C) {
    const size_t nchunks = (size_t)cdiv(HW, ST_ROWS), GBC = (size_t)G * B * C;
    return (nchunks * GBC * 2 + GBC * 2 + (size_t)G * B * 2) * sizeof(float);
}

extern "C" int cg_ln_stats(const float* y, float* mean, float* std, int G, int B, int HW, int C, void* ws, size_t ws_bytes,
                           void* stream) {
    if (int rc = check_c(C)) return rc;
    const long N = (long)HW * C;
    CG_REQUIRE(N > 1, "ln_stats: the unbiased std needs more than one element per sample (C*H*W = %ld)", N);
    const int nchunks = cdiv(HW, ST_ROWS);
    const size_t need = (size_t)nchunks * G * B * C * 2 * sizeof(float);
    if (need > ws_bytes) {
        set_error("ln_stats: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    launch_k(in_stats_partial_kernel, dim3(nchunks, G * B), 256, 0, st, y, (float*)ws, HW, C);
    if (int rc = check_launch("ln_stats_partial")) return rc;
    launch_k(ln_stats_final_kernel, G * B, LN_THREADS, 0, st, (const float*)ws, mean, std, G * B, C, nchunks, N);
    return check_launch("ln_stats_final");
}

extern "C" int cg_ln_act_fwd(const float* y, const float* mean, const float* std, const float* gamma, const float* beta, float eps,
                             float* z, int G, int B, int H, int W, int C, int act, void* stream) {
    if (int rc = check_c(C)) return rc;
    CG_REQUIRE(act == CG_ACT_NONE || act == CG_ACT_RELU || act == CG_ACT_LRELU, "ln_act_fwd: activation %d unsupported", act);
    CG_REQUIRE(gamma && beta, "ln_act_fwd: gamma and beta are required");
    NormP p{};
    p.y = y; p.mean = mean; p.rstd = std; p.ln_gamma = gamma; p.ln_beta = beta; p.ln_eps = eps; p.z = z;
    p.B = B; p.H = H; p.W = W; p.C = C; p.act = act;
    launch_k(norm_act_fwd_kernel<NM_LN>, dim3(cdiv((long)H * W, ST_ROWS), G * B), 256, 0, (cudaStream_t)stream, p);
    return check_launch("ln_act_fwd");
}

extern "C" int cg_ln_act_bwd(const float* dz, const float* y, const float* mean, const float* std, const float* gamma,
                             const float* beta, float eps, float* dy, float* dgamma, float* dbeta, int G, int B, int H, int W, int C,
                             int act, void* ws, size_t ws_bytes, void* stream) {
    if (int rc = check_c(C)) return rc;
    CG_REQUIRE(act == CG_ACT_NONE || act == CG_ACT_RELU || act == CG_ACT_LRELU, "ln_act_bwd: activation %d unsupported", act);
    CG_REQUIRE(gamma && beta && dgamma && dbeta, "ln_act_bwd: gamma, beta, dgamma and dbeta are required");
    const long N = (long)H * W * C;
    const int nchunks = cdiv((long)H * W, ST_ROWS);
    const long GBC = (long)G * B * C;
    const size_t need = cg_ln_workspace_bytes(G, B, H * W, C);
    if (need > ws_bytes) {
        set_error("ln_act_bwd: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    NormP p{};
    p.dz = dz; p.y = y; p.mean = mean; p.rstd = std; p.ln_gamma = gamma; p.ln_beta = beta; p.ln_eps = eps; p.dy = dy;
    p.B = B; p.H = H; p.W = W; p.C = C; p.act = act;
    p.part = (float*)ws;
    float* cs = p.part + (size_t)nchunks * GBC * 2;
    float* sums = cs + (size_t)GBC * 2;
    dim3 grid(nchunks, G * B);
    launch_k(norm_bwd_partial_kernel<NM_LN>, grid, 256, 0, st, p);
    if (int rc = check_launch("ln_bwd_partial")) return rc;
    launch_k(ln_bwd_final_kernel, G * B, LN_THREADS, 0, st, (const float*)p.part, gamma, std, cs, sums, G * B, B, C, nchunks, N);
    if (int rc = check_launch("ln_bwd_final")) return rc;
    launch_k(ln_param_grad_kernel, cdiv((long)G * C, 256), 256, 0, st, (const float*)cs, dgamma, dbeta, G, B, C);
    if (int rc = check_launch("ln_param_grad")) return rc;
    launch_k(norm_bwd_apply_kernel<NM_LN>, grid, 256, 0, st, p, (const float*)sums);
    return check_launch("ln_bwd_apply");
}
