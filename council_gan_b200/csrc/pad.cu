// Reflection padding of pad_type: reflect (Conv2dBlock, networks.py:470-471: nn.ReflectionPad2d(padding) followed by an nn.Conv2d with
// padding 0).  The TMA im2col fill of the tensor-core convolutions pads with zeros only, so a reflect layer reads a materialised padded
// copy of its input with pad 0; these are that copy and its backward.  Channels-last, member-stacked, one thread per pixel and 4 channels.
//
// Reference semantics (paths relative to the reference tree):
//   nn.ReflectionPad2d(p)             networks.py:470   index -i for i < 0 and 2 (n - 1) - i for i >= n: the edge pixel is not repeated
//   nn.Upsample(scale_factor=2)       networks.py:385   nearest, before the padding of the decoder's upsampling blocks
#include "common.cuh"

namespace cg {

__device__ __forceinline__ int reflect_index(int i, int n) {
    i = i < 0 ? -i : i;
    return i >= n ? 2 * (n - 1) - i : i;
}

// xp[n][Hs + 2p][Ws + 2p][C] = ReflectionPad2d(p) of x[n][H][W][C] seen at Hs x Ws = H x W, or 2H x 2W nearest-upsampled with ups
__global__ void reflect_pad_kernel(const float* __restrict__ x, float* __restrict__ xp, int H, int W, int C4, int p, int ups, int Hp,
                                   int Wp, long total) {
    pdl_trigger();
    pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = (int)(i % C4);
    long t = i / C4;
    const int ow = (int)(t % Wp);
    t /= Wp;
    const int oh = (int)(t % Hp);
    const long n = t / Hp;
    int h = reflect_index(oh - p, Hp - 2 * p), w = reflect_index(ow - p, Wp - 2 * p);
    h >>= ups;
    w >>= ups;
    reinterpret_cast<float4*>(xp)[i] = __ldg(reinterpret_cast<const float4*>(x) + ((n * H + h) * W + w) * C4 + c);
}

// the padded positions (0..3 of them: the pixel itself, and its mirror images above / below the edges when they fall inside the pad)
// that ReflectionPad2d(p) copies pixel h of a dimension of size n to, in ascending order
__device__ __forceinline__ int reflect_sources(int h, int n, int p, int* src) {
    int k = 0;
    if (h >= 1 && h <= p) src[k++] = p - h;              // mirrored above the first pixel
    src[k++] = p + h;
    if (h >= n - 1 - p && h <= n - 2) src[k++] = p + 2 * (n - 1) - h;  // mirrored below the last pixel
    return k;
}

// dx[n][H][W][C] = (fold(dxp) + addend) * act'(mask_src): every padded position of dxp[n][H + 2p][W + 2p][C] that reflects onto a pixel,
// summed row-major in padded order, then the addend, then the gate (as cg_conv_dgrad's epilogue applies them)
__global__ void reflect_pad_bwd_kernel(const float* __restrict__ dxp, float* __restrict__ dx, const float* __restrict__ addend,
                                       const float* __restrict__ mask_src, float slope, int H, int W, int C4, int p, long total) {
    pdl_trigger();
    pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = (int)(i % C4);
    long t = i / C4;
    const int w = (int)(t % W);
    t /= W;
    const int h = (int)(t % H);
    const long n = t / H;
    const int Hp = H + 2 * p, Wp = W + 2 * p;
    int rows[3], cols[3];
    const int nr = reflect_sources(h, H, p, rows), nc = reflect_sources(w, W, p, cols);
    const float4* src = reinterpret_cast<const float4*>(dxp) + n * Hp * Wp * C4 + c;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int a = 0; a < nr; ++a)
        for (int b = 0; b < nc; ++b) {
            const float4 v = __ldg(src + ((long)rows[a] * Wp + cols[b]) * C4);
            s.x += v.x;
            s.y += v.y;
            s.z += v.z;
            s.w += v.w;
        }
    if (addend) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(addend) + i);
        s.x += a.x;
        s.y += a.y;
        s.z += a.z;
        s.w += a.w;
    }
    if (mask_src) {
        const float4 m = __ldg(reinterpret_cast<const float4*>(mask_src) + i);
        s.x = m.x > 0.f ? s.x : s.x * slope;
        s.y = m.y > 0.f ? s.y : s.y * slope;
        s.z = m.z > 0.f ? s.z : s.z * slope;
        s.w = m.w > 0.f ? s.w : s.w * slope;
    }
    reinterpret_cast<float4*>(dx)[i] = s;
}

}  // namespace cg

using namespace cg;
#define ST ((cudaStream_t)stream)

extern "C" int cg_reflect_pad(const float* x, float* xp, int N, int H, int W, int C, int p, int ups, void* stream) {
    const int Hs = ups ? 2 * H : H, Ws = ups ? 2 * W : W;
    CG_REQUIRE(x && xp && N >= 1 && H >= 1 && W >= 1 && C >= 4 && C % 4 == 0 && (ups == 0 || ups == 1),
               "reflect_pad: N=%d H=%d W=%d C=%d ups=%d out of range", N, H, W, C, ups);
    CG_REQUIRE(p >= 1 && p < Hs && p < Ws, "reflect_pad: pad %d must be smaller than the padded map %dx%d", p, Hs, Ws);
    const int C4 = C / 4, Hp = Hs + 2 * p, Wp = Ws + 2 * p;
    const long total = (long)N * Hp * Wp * C4;
    launch_k(reflect_pad_kernel, cdiv(total, 256), 256, 0, ST, x, xp, H, W, C4, p, ups, Hp, Wp, total);
    return check_launch("reflect_pad");
}

extern "C" int cg_reflect_pad_bwd(const float* dxp, float* dx, const float* addend, const float* mask_src, float mask_slope, int N, int H,
                                  int W, int C, int p, void* stream) {
    CG_REQUIRE(dxp && dx && N >= 1 && H >= 1 && W >= 1 && C >= 4 && C % 4 == 0, "reflect_pad_bwd: N=%d H=%d W=%d C=%d out of range", N,
               H, W, C);
    CG_REQUIRE(p >= 1 && p < H && p < W, "reflect_pad_bwd: pad %d must be smaller than the map %dx%d", p, H, W);
    const int C4 = C / 4;
    const long total = (long)N * H * W * C4;
    launch_k(reflect_pad_bwd_kernel, cdiv(total, 256), 256, 0, ST, dxp, dx, addend, mask_src, mask_slope, H, W, C4, p, total);
    return check_launch("reflect_pad_bwd");
}
