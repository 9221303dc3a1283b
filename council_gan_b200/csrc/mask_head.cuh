// Attention-mask compositing of Decoder_V2_atten.forward (networks.py:398-407) and its backward, per pixel.  One copy shared by
// mask_head_fwd_kernel / mask_head_bwd_kernel (pointwise.cu) and the image reconstruction head (losses.cu), so that every kernel
// that composites produces the same bits: the sign the reconstruction backward takes comes from the value its forward summed.
#pragma once
#include "common.cuh"

namespace cg {

// h = tanh output of dec.model.9, 12 lanes: [o0 rgb | o1 rgb | o2 rgb | m0 m1 m2]
// mask_k = (tanh(10*h[9+k])+1)/2;  im[k+1] = (1-mask_k)*im[k] + mask_k*o_k, k = 0..2, im[0] = x_in; the output image is im[3]
struct MaskHeadPix {
    float hv[12], tk[3], mk[3], im[4][3];
};

__device__ __forceinline__ void mask_composite(const float* __restrict__ hp, const float* __restrict__ xp, MaskHeadPix& p) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(hp)), b = __ldg(reinterpret_cast<const float4*>(hp + 4)),
                 c = __ldg(reinterpret_cast<const float4*>(hp + 8));
    const float hv[12] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w};
#pragma unroll
    for (int j = 0; j < 12; j++) p.hv[j] = hv[j];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        p.tk[k] = tanhf(10.f * p.hv[9 + k]);
        p.mk[k] = (p.tk[k] + 1.f) * 0.5f;
    }
    const float4 xi = __ldg(reinterpret_cast<const float4*>(xp));
    p.im[0][0] = xi.x; p.im[0][1] = xi.y; p.im[0][2] = xi.z;
#pragma unroll
    for (int k = 0; k < 3; k++)
#pragma unroll
        for (int ch = 0; ch < 3; ch++) p.im[k + 1][ch] = (1.f - p.mk[k]) * p.im[k][ch] + p.mk[k] * p.hv[3 * k + ch];
}

// d(loss)/d(output image) dim (3 lanes, consumed) and d(loss)/d(mask) dm -> out[12] = d(loss)/d(pre-tanh output of dec.model.9)
__device__ __forceinline__ void mask_head_grad(const MaskHeadPix& p, float (&dim)[3], const float (&dm)[3], float (&out)[12]) {
    float dh[12];
#pragma unroll
    for (int k = 2; k >= 0; k--) {
        float dmk = dm[k];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
            dh[3 * k + ch] = p.mk[k] * dim[ch];
            dmk += dim[ch] * (p.hv[3 * k + ch] - p.im[k][ch]);
            dim[ch] *= (1.f - p.mk[k]);
        }
        dh[9 + k] = dmk * 5.f * (1.f - p.tk[k] * p.tk[k]);  // d/dh (tanh(10h)+1)/2
    }
#pragma unroll
    for (int j = 0; j < 12; j++) out[j] = dh[j] * (1.f - p.hv[j] * p.hv[j]);  // through the layer's own tanh
}

__device__ __forceinline__ void store12(float* __restrict__ op, const float (&v)[12]) {
    *reinterpret_cast<float4*>(op) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(op + 4) = make_float4(v[4], v[5], v[6], v[7]);
    *reinterpret_cast<float4*>(op + 8) = make_float4(v[8], v[9], v[10], v[11]);
}

}  // namespace cg
