// The decoder tail of a no-grad generator pass as ONE kernel (Decoder_V2_atten, networks.py:391-407):
//
//   AdaIN normalise + ReLU of the last 3x3 block  ->  1x1 64->64 + ReLU  ->  1x1 64->64 + ReLU  ->  1x1 64->12 + tanh
//   ->  attention-mask compositing with the input image  ->  x_fake, mask
//
// As separate launches every arrow is a round trip of a [G][B][256][256][64] fp32 map (537 MB at the BASELINE shape) through
// HBM: norm_act_fwd 0.39 + two 1x1 convolutions 0.24 each + the 12-channel head 0.13 + mask head 0.05 ms = 1.05 ms per decoder
// pass, three such passes per iteration (dis_update, dis_council_update x2; the pass of gen_update keeps its activations for the
// backward and stays unfused).  Fused, the 64-channel map is read once and 8 floats per pixel are written.
//
// One CTA = 128 threads = one warpgroup = 128 pixels per tile, three co-resident CTAs per SM hide each other's latencies.  All
// threads gather / transform the tile into the K-major 128-byte-swizzled shared-memory operand (TF32-rounded), the warpgroup
// issues the wgmma MMAs (two 64-row halves, accumulators in registers), applies bias + ReLU and writes the next layer's operand
// into the same shared-memory tile.  The three weight matrices of the CTA's council member stay resident.
#include "common.cuh"
#include "tc_ptx.cuh"

namespace cg {

struct HeadP {
    const float* y; const float* mean; const float* rstd; const float* adain;
    const float* w1; const float* b1; const float* w2; const float* b2; const float* w3; const float* b3;
    const float* x_img; float* x_fake; float* mask;
    int G, B, HW, P, off, cpg;
};

constexpr int HD_THREADS = 128;
constexpr int HD_A = 32768;   // activation tile: 2 chunks of [128 rows x 128 B]
constexpr int HD_W = 16384;   // 64x64 weight matrix: 2 chunks of [64 rows x 128 B]
constexpr int HD_W3 = 4096;   // 16x64 (12 used): 2 chunks of [16 rows x 128 B]

__device__ __forceinline__ float4 hd_ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// rows x 64 K-major matrix (row stride 64 floats in global) -> chunk j = k / 32: [rows][128 B], 16-byte unit u at u ^ (row % 8)
__device__ __forceinline__ void stage_weights(uint8_t* dst, const float* w, int rows, int rows_pad) {
    for (int i = threadIdx.x; i < 2 * rows_pad * 8; i += HD_THREADS) {
        const int u = i & 7, r = (i >> 3) % rows_pad, j = i / (8 * rows_pad);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < rows) v = to_tf32(hd_ldg4(w + (long)r * 64 + j * 32 + u * 4));
        *reinterpret_cast<float4*>(dst + j * (rows_pad * 128) + (r >> 3) * 1024 + (r & 7) * 128 + ((u ^ (r & 7)) << 4)) = v;
    }
}

__global__ void __launch_bounds__(HD_THREADS, 3) head_fused_kernel(const HeadP p) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* sA = smem;
    uint8_t* sW1 = sA + HD_A;
    uint8_t* sW2 = sW1 + HD_W;
    uint8_t* sW3 = sW2 + HD_W;
    float* s_b1 = reinterpret_cast<float*>(sW3 + HD_W3);  // 64
    float* s_b2 = s_b1 + 64;                               // 64
    float* s_b3 = s_b2 + 64;                               // 16

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = blockIdx.x % p.G, cidx = blockIdx.x / p.G;
    const int tiles = (int)(((long)p.B * p.HW) >> 7);

    stage_weights(sW1, p.w1 + (long)g * 64 * 64, 64, 64);
    stage_weights(sW2, p.w2 + (long)g * 64 * 64, 64, 64);
    stage_weights(sW3, p.w3 + (long)g * 12 * 64, 12, 16);
    if (threadIdx.x < 64) {
        s_b1[threadIdx.x] = __ldg(p.b1 + g * 64 + threadIdx.x);
        s_b2[threadIdx.x] = __ldg(p.b2 + g * 64 + threadIdx.x);
    }
    if (threadIdx.x < 16) s_b3[threadIdx.x] = threadIdx.x < 12 ? __ldg(p.b3 + g * 12 + threadIdx.x) : 0.f;
    const uint64_t desc_hi = make_kmajor_sw128_desc(0);
    const uint32_t a_addr = smem_u32(sA);

    // loader mapping (coalesced: 8 threads read one 128-byte line): 16-byte unit u of rows r0, r0 + 16, ...
    const int u = threadIdx.x & 7, r0 = threadIdx.x >> 3;
    // accumulator mapping (wgmma): rows 64 h + 16 warp + lane / 4 (+ 8) of half h, columns 8 j + 2 (lane % 4) (+ 1)
    const int arow = warp * 16 + (lane >> 2), acol = 2 * (lane & 3);
    const int row = threadIdx.x;  // pixel row of the mask head
    float acc[2][32];
    float hacc[2][8];

    // D[128 x N] = A[128 x 64] * W^T: K = 64 = 2 chunks x 4 steps of 8, for both 64-row halves of the tile
    auto issue64 = [&](uint32_t w_addr) {
        fence_proxy_async();
        __syncthreads();
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int q = 0; q < 8; q++) {
                const int j = q >> 2, kk = q & 3;
                const uint64_t adesc = (desc_hi | (uint64_t)(((a_addr + j * 16384 + h * 8192) & 0x3FFFF) >> 4)) + (uint64_t)(kk * 2);
                const uint64_t bdesc = (desc_hi | (uint64_t)(((w_addr + j * 8192) & 0x3FFFF) >> 4)) + (uint64_t)(kk * 2);
                wgmma_tf32<64>(acc[h], adesc, bdesc, q != 0 ? 1 : 0);
            }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_reg_fence(acc[0], 32);
        wgmma_reg_fence(acc[1], 32);
        __syncthreads();  // every MMA reading the tile has retired before it is overwritten
    };
    // accumulator + bias, ReLU, TF32 -> the shared-memory operand of the next layer
    auto relayer = [&](const float* bias) {
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int r = h * 64 + arow + 8 * e;
                uint8_t* dst = sA + (r >> 3) * 1024 + (r & 7) * 128;
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const int c = 8 * j + acol;
                    float2 o;
                    o.x = to_tf32(fmaxf(acc[h][4 * j + 2 * e] + bias[c], 0.f));
                    o.y = to_tf32(fmaxf(acc[h][4 * j + 2 * e + 1] + bias[c + 1], 0.f));
                    *reinterpret_cast<float2*>(dst + (c >> 5) * 16384 + ((((c & 31) >> 2) ^ (r & 7)) << 4) + (c & 3) * 4) = o;
                }
            }
    };

    for (int tile = cidx; tile < tiles; tile += p.cpg) {
        const long m0 = (long)tile * 128;        // first pixel of the tile within the member (B * HW pixels)
        const int img = (int)(m0 / p.HW);        // HW % 128 == 0: a tile lies inside one image
        const long gb = (long)g * p.B + img;
        // ---- AdaIN affine of this thread's 8 channels (c = j * 32 + u * 4 .. + 3), then gather + transform the tile
        float4 a[2], b[2];
#pragma unroll
        for (int j = 0; j < 2; j++) {
            const int c = j * 32 + u * 4;
            const float4 mu = hd_ldg4(p.mean + gb * 64 + c), rs = hd_ldg4(p.rstd + gb * 64 + c);
            float4 ga = make_float4(1.f, 1.f, 1.f, 1.f), be = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p.adain) {
                const float* ap = p.adain + gb * p.P + p.off;
                be = hd_ldg4(ap + c);
                ga = hd_ldg4(ap + 64 + c);
            }
            a[j] = make_float4(ga.x * rs.x, ga.y * rs.y, ga.z * rs.z, ga.w * rs.w);
            b[j] = make_float4(be.x - mu.x * a[j].x, be.y - mu.y * a[j].y, be.z - mu.z * a[j].z, be.w - mu.w * a[j].w);
        }
        const float* yb = p.y + ((long)g * p.B * p.HW + m0) * 64 + u * 4;
        float4 v[16];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            v[2 * i] = hd_ldg4(yb + (long)(r0 + 16 * i) * 64);
            v[2 * i + 1] = hd_ldg4(yb + (long)(r0 + 16 * i) * 64 + 32);
        }
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int r = r0 + 16 * i;
            uint8_t* dst = sA + (r >> 3) * 1024 + (r & 7) * 128 + ((u ^ (r & 7)) << 4);
#pragma unroll
            for (int j = 0; j < 2; j++) {
                const float4 x = v[2 * i + j];
                float4 o;
                o.x = fmaxf(fmaf(x.x, a[j].x, b[j].x), 0.f);
                o.y = fmaxf(fmaf(x.y, a[j].y, b[j].y), 0.f);
                o.z = fmaxf(fmaf(x.z, a[j].z, b[j].z), 0.f);
                o.w = fmaxf(fmaf(x.w, a[j].w, b[j].w), 0.f);
                *reinterpret_cast<float4*>(dst + j * 16384) = to_tf32(o);
            }
        }
        issue64(smem_u32(sW1));   // dec.model.7: 1x1 64->64
        relayer(s_b1);
        issue64(smem_u32(sW2));   // dec.model.8: 1x1 64->64
        relayer(s_b2);
        // dec.model.9: 1x1 64->12 (N padded to 16), tanh below
        fence_proxy_async();
        __syncthreads();
        wgmma_fence();
#pragma unroll
        for (int hh = 0; hh < 2; hh++)
#pragma unroll
            for (int q = 0; q < 8; q++) {
                const int j = q >> 2, kk = q & 3;
                const uint64_t adesc = (desc_hi | (uint64_t)(((a_addr + j * 16384 + hh * 8192) & 0x3FFFF) >> 4)) + (uint64_t)(kk * 2);
                const uint64_t bdesc = (desc_hi | (uint64_t)(((smem_u32(sW3) + j * 2048) & 0x3FFFF) >> 4)) + (uint64_t)(kk * 2);
                wgmma_tf32<16>(hacc[hh], adesc, bdesc, q != 0 ? 1 : 0);
            }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_reg_fence(hacc[0], 8);
        wgmma_reg_fence(hacc[1], 8);
        __syncthreads();
        // the 16 head columns of a pixel are spread over four lanes: regroup them per row through the (now free) tile
        float* s_h = reinterpret_cast<float*>(sA);  // [128][17]
#pragma unroll
        for (int hh = 0; hh < 2; hh++)
#pragma unroll
            for (int e = 0; e < 2; e++)
#pragma unroll
                for (int j = 0; j < 2; j++) {
                    const int r = hh * 64 + arow + 8 * e;
                    s_h[r * 17 + 8 * j + acol] = hacc[hh][4 * j + 2 * e];
                    s_h[r * 17 + 8 * j + acol + 1] = hacc[hh][4 * j + 2 * e + 1];
                }
        __syncthreads();
        // ---- mask head (networks.py:398-407): h = tanh(.), [o0 rgb | o1 rgb | o2 rgb | m0 m1 m2]
        float h[12];
#pragma unroll
        for (int j = 0; j < 12; j++) h[j] = tanhf(s_h[row * 17 + j] + s_b3[j]);
        const long pix = m0 + row;                       // pixel within the member
        const float4 xi = hd_ldg4(p.x_img + (pix % ((long)p.B * p.HW)) * 4);
        float im[3] = {xi.x, xi.y, xi.z};
        float mk[3];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            mk[k] = (tanhf(10.f * h[9 + k]) + 1.f) * 0.5f;
#pragma unroll
            for (int ch = 0; ch < 3; ch++) im[ch] = (1.f - mk[k]) * im[ch] + mk[k] * h[3 * k + ch];
        }
        const long o = ((long)g * p.B * p.HW + pix) * 4;
        *reinterpret_cast<float4*>(p.x_fake + o) = make_float4(im[0], im[1], im[2], 0.f);
        *reinterpret_cast<float4*>(p.mask + o) = make_float4(mk[0], mk[1], mk[2], 0.f);
        __syncthreads();  // the next tile's gather overwrites the regrouped head outputs
    }
}

}  // namespace cg

using namespace cg;

extern "C" int cg_head_fused(const float* y, const float* mean, const float* rstd, const float* adain, int P, int off, const float* w1,
                             const float* b1, const float* w2, const float* b2, const float* w3, const float* b3, const float* x_img,
                             float* x_fake, float* mask, int G, int B, int HW, void* stream) {
    CG_REQUIRE(G >= 1 && B >= 1 && HW % 128 == 0, "head_fused: needs H*W %% 128 == 0 (got %d)", HW);
    const int sms = tc_sm_count();
    CG_REQUIRE(sms > 0 && G <= 3 * sms, "head_fused: no device / too many groups");
    HeadP p{};
    p.y = y; p.mean = mean; p.rstd = rstd; p.adain = adain; p.w1 = w1; p.b1 = b1; p.w2 = w2; p.b2 = b2; p.w3 = w3; p.b3 = b3;
    p.x_img = x_img; p.x_fake = x_fake; p.mask = mask; p.G = G; p.B = B; p.HW = HW; p.P = P; p.off = off;
    p.cpg = 3 * sms / G;
    const long tiles = (long)B * HW / 128;
    if (p.cpg > tiles) p.cpg = (int)tiles;
    const size_t smem = HD_A + 2 * HD_W + HD_W3 + (64 + 64 + 16) * 4 + 1024;
    static PerDeviceOnce attr_once;
    if (attr_once.first()) {
        cudaError_t e = cudaFuncSetAttribute(head_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) {
            set_error("cudaFuncSetAttribute(head_fused_kernel): %s", cudaGetErrorString(e));
            return CG_ERR_CUDA;
        }
    }
    launch_k(head_fused_kernel, G * p.cpg, HD_THREADS, smem, (cudaStream_t)stream, p);
    return check_launch("head_fused");
}
