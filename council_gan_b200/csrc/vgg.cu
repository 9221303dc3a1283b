// The frozen VGG-16 of the perceptual loss vgg_w (trainer_council.py:199-205, 531-538, 636-641): its input preprocessing and the
// 2x2 max-pools between its convolution stages, forward and data gradient.  The 3x3 convolutions run on cg_conv_fwd / cg_conv_dgrad
// and the loss itself (instance-normalised squared error of relu5_3) is cg_vgg_loss in losses.cu.
//
// Reference semantics (paths relative to the reference tree):
//   vgg_preprocess                     utils.py:380-390     RGB -> BGR, (x + 1) * 255 * 0.5, minus the BGR mean
//   Vgg16.forward                      networks.py:594-622  F.max_pool2d(h, kernel_size=2, stride=2) after conv1_2, conv2_2, conv3_3
#include "common.cuh"

namespace cg {

// vgg_preprocess on channels-last pixels [npix][4] (lanes 0..2 = RGB): y = {B', G', R', 0} with c' = (x_c + 1) * 255 * 0.5 - mean_c,
// each operation rounded as torch rounds it (no contraction into an FMA)
__global__ void vgg_preprocess_kernel(const float* __restrict__ x, float* __restrict__ y, long npix) {
    pdl_trigger();
    pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    auto f = [](float c, float mean) { return __fsub_rn(__fmul_rn(__fmul_rn(__fadd_rn(c, 1.f), 255.f), 0.5f), mean); };
    reinterpret_cast<float4*>(y)[i] = make_float4(f(v.z, 103.939f), f(v.y, 116.779f), f(v.x, 123.680f), 0.f);
}

// its data gradient: d_x[c] (+)= 127.5 * dy[2 - c] on lanes 0..2; lane 3 is written 0 (accumulate 0) or kept (accumulate 1)
__global__ void vgg_preprocess_bwd_kernel(const float* __restrict__ dy, float* __restrict__ d_x, long npix, int accumulate) {
    pdl_trigger();
    pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npix) return;
    const float4 g = __ldg(reinterpret_cast<const float4*>(dy) + i);
    float4* o = reinterpret_cast<float4*>(d_x) + i;
    float4 r = accumulate ? *o : make_float4(0.f, 0.f, 0.f, 0.f);
    r.x = __fadd_rn(r.x, __fmul_rn(127.5f, g.z));  // rounded twice, as autograd's product and the accumulating add are
    r.y = __fadd_rn(r.y, __fmul_rn(127.5f, g.y));
    r.z = __fadd_rn(r.z, __fmul_rn(127.5f, g.x));
    *o = r;
}

// max_pool2d(2, 2), floor size: one thread per output pixel and 4 channels.  x [N][H][W][C] -> y [N][H/2][W/2][C]
__global__ void maxpool2x2_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W, int C4, int Ho, int Wo,
                                      long total) {
    pdl_trigger();
    pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = (int)(i % C4);
    long t = i / C4;
    const int wo = (int)(t % Wo);
    t /= Wo;
    const int ho = (int)(t % Ho);
    const long n = t / Ho;
    const float4* xp = reinterpret_cast<const float4*>(x) + ((n * H + 2 * ho) * W + 2 * wo) * C4 + c;
    const float4 a = __ldg(xp), b = __ldg(xp + C4), d = __ldg(xp + (long)W * C4), e = __ldg(xp + (long)W * C4 + C4);
    reinterpret_cast<float4*>(y)[i] = make_float4(fmaxf(fmaxf(a.x, b.x), fmaxf(d.x, e.x)), fmaxf(fmaxf(a.y, b.y), fmaxf(d.y, e.y)),
                                                  fmaxf(fmaxf(a.z, b.z), fmaxf(d.z, e.z)), fmaxf(fmaxf(a.w, b.w), fmaxf(d.w, e.w)));
}

// position (0..3, row-major) of the first maximum of a 2x2 window, as max_pool2d picks it (a later value must be strictly greater)
__device__ __forceinline__ int argmax4(float v0, float v1, float v2, float v3) {
    int k = 0;
    float m = v0;
    if (v1 > m) { m = v1; k = 1; }
    if (v2 > m) { m = v2; k = 2; }
    if (v3 > m) k = 3;
    return k;
}

// backward of max_pool2d(relu(pre)) w.r.t. pre, with no index tensor: one thread per INPUT pixel and 4 channels recomputes its
// window's argmax from x (the saved ReLU output) and takes dy where it is that argmax and x > 0; every other position, and the last
// row / column that an odd size leaves uncovered, gets 0.  dx [N][H][W][C], dy [N][H/2][W/2][C]
__global__ void maxpool2x2_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ dx, int H, int W,
                                      int C4, int Ho, int Wo, long total) {
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
    const int ho = h >> 1, wo = w >> 1;
    float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
    if (ho < Ho && wo < Wo) {
        const float4* xp = reinterpret_cast<const float4*>(x) + ((n * H + 2 * ho) * W + 2 * wo) * C4 + c;
        const float4 a = __ldg(xp), b = __ldg(xp + C4), d = __ldg(xp + (long)W * C4), e = __ldg(xp + (long)W * C4 + C4);
        const int mine = (h & 1) * 2 + (w & 1);
        const float4 self = mine == 0 ? a : mine == 1 ? b : mine == 2 ? d : e;
        const float4 g = __ldg(reinterpret_cast<const float4*>(dy) + ((n * Ho + ho) * Wo + wo) * C4 + c);
        r.x = argmax4(a.x, b.x, d.x, e.x) == mine && self.x > 0.f ? g.x : 0.f;
        r.y = argmax4(a.y, b.y, d.y, e.y) == mine && self.y > 0.f ? g.y : 0.f;
        r.z = argmax4(a.z, b.z, d.z, e.z) == mine && self.z > 0.f ? g.z : 0.f;
        r.w = argmax4(a.w, b.w, d.w, e.w) == mine && self.w > 0.f ? g.w : 0.f;
    }
    reinterpret_cast<float4*>(dx)[i] = r;
}

}  // namespace cg

using namespace cg;
#define ST ((cudaStream_t)stream)

extern "C" int cg_vgg_preprocess(const float* x, float* y, long npix, void* stream) {
    CG_REQUIRE(x && y && npix >= 1, "vgg_preprocess: npix=%ld out of range", npix);
    launch_k(vgg_preprocess_kernel, cdiv(npix, 256), 256, 0, ST, x, y, npix);
    return check_launch("vgg_preprocess");
}

extern "C" int cg_vgg_preprocess_bwd(const float* dy, float* d_x, long npix, int accumulate, void* stream) {
    CG_REQUIRE(dy && d_x && npix >= 1, "vgg_preprocess_bwd: npix=%ld out of range", npix);
    launch_k(vgg_preprocess_bwd_kernel, cdiv(npix, 256), 256, 0, ST, dy, d_x, npix, accumulate);
    return check_launch("vgg_preprocess_bwd");
}

extern "C" int cg_maxpool2x2_fwd(const float* x, float* y, int N, int H, int W, int C, void* stream) {
    CG_REQUIRE(x && y && N >= 1 && H >= 2 && W >= 2 && C >= 4 && C % 4 == 0, "maxpool2x2_fwd: N=%d H=%d W=%d C=%d out of range", N, H,
               W, C);
    const int Ho = H / 2, Wo = W / 2, C4 = C / 4;
    const long total = (long)N * Ho * Wo * C4;
    launch_k(maxpool2x2_fwd_kernel, cdiv(total, 256), 256, 0, ST, x, y, H, W, C4, Ho, Wo, total);
    return check_launch("maxpool2x2_fwd");
}

extern "C" int cg_maxpool2x2_bwd(const float* dy, const float* x, float* dx, int N, int H, int W, int C, void* stream) {
    CG_REQUIRE(dy && x && dx && N >= 1 && H >= 2 && W >= 2 && C >= 4 && C % 4 == 0, "maxpool2x2_bwd: N=%d H=%d W=%d C=%d out of range",
               N, H, W, C);
    const int C4 = C / 4;
    const long total = (long)N * H * W * C4;
    launch_k(maxpool2x2_bwd_kernel, cdiv(total, 256), 256, 0, ST, dy, x, dx, H, W, C4, H / 2, W / 2, total);
    return check_launch("maxpool2x2_bwd");
}
