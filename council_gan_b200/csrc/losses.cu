// Fused loss kernels of the three updates (SURVEY K12-K14): LSGAN over every discriminator scale, the focus
// losses, the loss-history matching and all their gradients -- 1 launch per discriminator update and direction,
// 2 launches per gen_update and direction (a reduction pass, then -- after the data-parallel all-reduce of the 6N
// scalars -- one pass that finalises the loss values ON THE DEVICE and writes every gradient).  No host round trip.
//
// Reference semantics (paths relative to the reference tree):
//   MsImageDis.calc_dis_loss / calc_gen_loss                networks.py:56-64, 84-90   (lsgan)
//   MsImageDisCouncil.calc_dis_loss / calc_gen_loss         networks.py:158-166, 188-194
//   mask_zero_one_criterion / mask_small_criterion(_square) / mask_criterion_TV   trainer_council.py:230-250
//   loss-history matching                                   trainer_council.py:518-524, 576-586
//   total-loss assembly in gen_update                       trainer_council.py:392-451, 497-529, 559-634
//   abs_beginning_end (recon_criterion_v2_color)            trainer_council.py:210-215, 477-495  (2 more launches per direction
//                                                           while its weight gate is open)
//   recon_x (recon_criterion of the within-domain decode)   trainer_council.py:339-345, 455-459
//   council_abs_w (council_basic_criterion_*)               trainer_council.py:224-228, 595-619  (2 more launches per direction
//                                                           while the council gate is open)
//   vgg_w (compute_vgg_loss on relu5_3)                     trainer_council.py:531-538, 636-641  (1 launch per update)
#include "common.cuh"
#include "mask_head.cuh"

namespace cg {

__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float sgnf(float x) { return (float)((x > 0.f) - (x < 0.f)); }

template <int N>
__device__ __forceinline__ void block_sum(float (&v)[N], float* smem /* >= N*32 */) {
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

// "last block done" ticket: returns true in exactly one block (all threads), after every other block's partials are visible.
__device__ __forceinline__ bool last_block_done(unsigned int* counter, unsigned int nblocks) {
    __shared__ unsigned int s_ticket;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_ticket = atomicAdd(counter, 1u);
    __syncthreads();
    bool last = s_ticket == nblocks - 1;
    if (last) __threadfence();
    return last;
}

// ---------------------------------------------------------------------------------------------------------------
// discriminator updates: LSGAN loss of every scale + its gradient, one launch
// ---------------------------------------------------------------------------------------------------------------
// block b -> (map m, member g, segment s); ws: float part[nmaps][G][nseg] then the ticket counter
__global__ void __launch_bounds__(256) lsgan_fused_kernel(const cg_lsgan_desc d, float* __restrict__ loss_total, int accumulate,
                                                          float* __restrict__ loss_plain, float* __restrict__ part,
                                                          unsigned int* __restrict__ counter) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sm[32];
    const int nseg = d.nseg, G = d.G;
    int b = blockIdx.x;
    const int m = b / (G * nseg);
    b -= m * G * nseg;
    const int g = b / nseg, s = b - g * nseg;
    const int n = d.n_per_seg[m];
    const float t = d.target[s];
    const float coef = d.grad_scale * d.weight[g][s] * 2.0f / (float)n;
    const float* p = d.out[m] + ((long)g * nseg + s) * n;
    float* q = d.dout[m] ? d.dout[m] + ((long)g * nseg + s) * n : nullptr;
    float v[1] = {0.f};
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        float df = __ldg(p + i) - t;
        v[0] += df * df;
        if (q) q[i] = coef * df;
    }
    block_sum<1>(v, sm);
    if (threadIdx.x == 0) part[(m * G + g) * nseg + s] = v[0];
    if (!last_block_done(counter, gridDim.x)) return;
    if (threadIdx.x < G) {
        const int gg = threadIdx.x;
        const volatile float* vp = part;
        float tot = 0.f, plain = 0.f;
        for (int mm = 0; mm < d.nmaps; mm++) {
            float tm = 0.f, pm = 0.f;
            for (int ss = 0; ss < nseg; ss++) {
                float mean = vp[(mm * G + gg) * nseg + ss] / (float)d.n_per_seg[mm];
                tm += d.weight[gg][ss] * mean;
                pm += mean;
            }
            tot += tm;
            plain += pm;
        }
        tot *= d.loss_scale;
        loss_total[gg] = accumulate ? loss_total[gg] + tot : tot;
        if (loss_plain) loss_plain[gg] = plain * d.loss_scale;
    }
    if (threadIdx.x == 0) *counter = 0u;
}

// ---------------------------------------------------------------------------------------------------------------
// gen_update, pass 1: every reduction of the generator loss in one launch
// ---------------------------------------------------------------------------------------------------------------
constexpr int GL_PIX = 2048;  // mask pixels per focus block

// blocks [0, nmaps*G): LSGAN maps (adversarial D maps first, then council-D maps); then nchunks*G focus blocks.
// ws: float part_map[nmaps][G]; float part_focus[nchunks][G][4]; ticket counter.
__global__ void __launch_bounds__(256) gen_loss_fwd_kernel(const cg_gen_loss_desc d, float* __restrict__ scal, float* __restrict__ part_map,
                                                           float* __restrict__ part_focus, unsigned int* __restrict__ counter, int nchunks) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sm[4 * 32];
    const int G = d.G, nmaps = d.n_adv + d.n_cl;
    const int b = blockIdx.x;
    if (b < nmaps * G) {
        const int m = b / G, g = b - m * G;
        const bool adv = m < d.n_adv;
        const int n = adv ? d.adv_n[m] : d.cl_n[m - d.n_adv];
        const float* p = (adv ? d.adv_out[m] : d.cl_out[m - d.n_adv]) + (long)g * n;
        float* q = adv && d.adv_dout[m] ? d.adv_dout[m] + (long)g * n : nullptr;
        const float coef = d.adv_grad_scale * 2.0f / (float)n;
        float v[1] = {0.f};
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            float df = __ldg(p + i) - 1.0f;  // calc_gen_loss: target 1 (networks.py:90,194)
            v[0] += df * df;
            if (q) q[i] = coef * df;
        }
        block_sum<1>(v, sm);
        if (threadIdx.x == 0) part_map[m * G + g] = v[0];
    } else {
        const int fb = b - nmaps * G;
        const int g = fb % G, chunk = fb / G;
        const int H = d.H, W = d.W;
        const long npix = (long)d.B * H * W;
        const long p0 = (long)chunk * GL_PIX, p1 = min(npix, p0 + GL_PIX);
        const float* mb = d.mask + (long)g * npix * 4;
        const float center = d.center, eps = d.eps;
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        for (long px = p0 + threadIdx.x; px < p1; px += blockDim.x) {
            int w = (int)(px % W);
            int h = (int)((px / W) % H);
            float4 mk = ld4(mb + px * 4);
            v[0] += 1.f / (fabsf(mk.x - center) + eps) + 1.f / (fabsf(mk.y - center) + eps) + 1.f / (fabsf(mk.z - center) + eps);
            v[1] += mk.x + mk.y + mk.z;
            if (h + 1 < H) {
                float4 q = ld4(mb + (px + W) * 4);
                v[2] += fabsf(q.x - mk.x) + fabsf(q.y - mk.y) + fabsf(q.z - mk.z);
            }
            if (w + 1 < W) {
                float4 r = ld4(mb + (px + 1) * 4);
                v[3] += fabsf(r.x - mk.x) + fabsf(r.y - mk.y) + fabsf(r.z - mk.z);
            }
        }
        block_sum<4>(v, sm);
        if (threadIdx.x == 0) {
            float* o = part_focus + ((long)chunk * G + g) * 4;
            o[0] = v[0]; o[1] = v[1]; o[2] = v[2]; o[3] = v[3];
        }
    }
    if (!last_block_done(counter, gridDim.x)) return;
    // scal[g] = { sum_scales mean (D(x)-1)^2, sum_scales mean (DC(x)-1)^2, focus sums[4] }   (local to this rank)
    const int t = threadIdx.x;
    if (t < G * 6) {
        const int g = t / 6, k = t - g * 6;
        float r = 0.f;
        if (k < 2) {
            const volatile float* vp = part_map;
            int m0 = k == 0 ? 0 : d.n_adv, m1 = k == 0 ? d.n_adv : nmaps;
            for (int m = m0; m < m1; m++) {
                int n = m < d.n_adv ? d.adv_n[m] : d.cl_n[m - d.n_adv];
                r += vp[m * G + g] / (float)n;
            }
        } else if (d.mask) {
            const volatile float* vp = part_focus;
            double s = 0.0;
            for (int c = 0; c < nchunks; c++) s += (double)vp[((long)c * G + g) * 4 + (k - 2)];
            r = (float)s;
        }
        scal[g * 6 + k] = r;
    }
    if (t == 0) *counter = 0u;
}

// ---------------------------------------------------------------------------------------------------------------
// gen_update, pass 2: finalise the loss values on the device, then every remaining gradient, one launch
// ---------------------------------------------------------------------------------------------------------------
struct GenCoef {      // per member, computed redundantly by every block
    float cdis;       // council-loss weight of this member: w_match * council_w          (gradient of DC maps)
    float c01, csum, ctv;  // focus-loss gradient coefficients
};

// hist rings: double [G][hist+1]; the live window is positions (head+k) % (hist+1), k = 0..hist-1; an append writes
// position (head+hist) % (hist+1) (not in anybody's read set) and the HOST advances head afterwards.
__device__ __forceinline__ double ring_mean_after_append(const double* ring, int R, int head, int hist, double v, int lane) {
    double s = 0.0;
    for (int k = 1 + lane; k < hist; k += 32) s += ring[(head + k) % R];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return (s + v) / (double)hist;
}
__device__ __forceinline__ double ring_mean(const double* ring, int R, int head, int hist, int lane) {
    double s = 0.0;
    for (int k = lane; k < hist; k += 32) s += ring[(head + k) % R];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s / (double)hist;
}

__global__ void __launch_bounds__(256) gen_loss_bwd_kernel(const cg_gen_loss_desc d, const cg_gen_loss_hp hp, const float* __restrict__ scal,
                                                           double* __restrict__ hist_gan, double* __restrict__ hist_council,
                                                           float* __restrict__ total, double* __restrict__ total64, int accumulate,
                                                           float* __restrict__ pub, float* __restrict__ d_mask, int map_blocks) {
    pdl_trigger();
    pdl_wait();
    __shared__ GenCoef sc[CG_LOSS_MAX_G];
    const int G = d.G;
    const int R = hp.hist_size + 1;
    // ---- finalise (warp 0 of every block; block 0 also publishes and appends to the histories) --------------------
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        for (int g = 0; g < G; g++) {
            const double adv = (double)scal[g * 6 + 0] / (double)hp.world;  // mean over the GLOBAL minibatch (equal shards)
            const double cl = (double)scal[g * 6 + 1] / (double)hp.world;
            const double l01 = (double)scal[g * 6 + 2] / hp.numel;
            const double msum = (double)scal[g * 6 + 3] / hp.numel;
            const double ltv = ((double)scal[g * 6 + 4] + (double)scal[g * 6 + 5]) / hp.numel;
            double tot = 0.0, ltot = 0.0, c01 = 0.0, csum = 0.0, ctv = 0.0;
            const double* rg = hist_gan + (long)g * R;
            const bool fm = hp.focus_on && hp.focus_matching;
            // focus matching (:398-410, 433-445) runs before the GAN block: its ratios read the GAN history before this append
            const double gan_before = fm ? ring_mean(rg, R, hp.head_gan, hp.hist_size, lane) : 1.0;
            double w01m = 1.0, wtm = 1.0, l01_32 = 0.0, ltot_app = 0.0;
            if (hp.focus_on) {
                if (hp.w01 != 0.0) {                                                             // trainer_council.py:392-415
                    double s01 = 1.0;
                    if (fm) {  // append the unscaled float32 term, then scale it in place by the float32 ratio
                        l01_32 = (double)(float)l01;
                        w01m = gan_before / ring_mean_after_append(hp.hist_focus01 + (long)g * R, R, hp.head_focus01, hp.hist_size, l01_32, lane);
                        s01 = (double)(float)w01m;
                    }
                    tot += hp.w01 * l01 * s01;
                    c01 = hp.w01 * s01 / hp.numel;
                }
                if (hp.wtv != 0.0) { tot += hp.wtv * ltv; ctv = hp.wtv / hp.numel; }            // :425-431 (never matched)
                if (hp.wtot != 0.0) {                                                            // :418-422, :447-451
                    if (hp.small_abs) { ltot += fabs(msum); csum += hp.wtot * (double)((msum > 0.0) - (msum < 0.0)) / hp.numel; }
                    if (hp.small_square) { ltot += msum * msum; csum += hp.wtot * 2.0 * msum / hp.numel; }
                    if (fm) {  // b2a appends a2b's scaled term (:441), a2b its own unscaled one (:435)
                        ltot_app = hp.focus_src ? (double)hp.focus_src[g * 8 + 3] : (double)(float)ltot;
                        wtm = gan_before / ring_mean_after_append(hp.hist_focus + (long)g * R, R, hp.head_focus, hp.hist_size, ltot_app, lane);
                        ltot *= (double)(float)wtm;
                        csum *= (double)(float)wtm;
                    }
                    tot += hp.wtot * ltot;
                }
            }
            double mean_gan;
            const double adv32 = (double)(float)adv;  // the history stores the float32 loss value (:520)
            if (hp.gan_on) {
                mean_gan = hp.matching ? ring_mean_after_append(rg, R, hp.head_gan, hp.hist_size, adv32, lane)
                                       : ring_mean(rg, R, hp.head_gan, hp.hist_size, lane);
                tot += hp.gan_w * adv;
            } else {
                mean_gan = ring_mean(rg, R, hp.head_gan, hp.hist_size, lane);
            }
            double w = 1.0, closs = 0.0, cdis = 0.0;
            if (hp.council_on) {
                if (hp.matching) {  // :576-586
                    const double cl32 = (double)(float)cl;
                    double mean_c = ring_mean_after_append(hist_council + (long)g * R, R, hp.head_council, hp.hist_size, cl32, lane);
                    w = mean_gan / mean_c;
                }
                closs = cl * (double)(float)w * hp.council_w;  // float32 tensor * python float (cast to float32) * council_w
                tot += closs;
                cdis = w * hp.council_w;
            }
            if (lane == 0) {
                sc[g].cdis = (float)cdis;
                sc[g].c01 = (float)c01;
                sc[g].csum = (float)csum;
                sc[g].ctv = (float)ctv;
                if (blockIdx.x == 0) {
                    double t64 = accumulate ? total64[g] + tot : tot;  // directions are summed in double, published as float32
                    total64[g] = t64;
                    total[g] = (float)t64;
                    float* o = pub + g * 8;
                    o[0] = (float)tot; o[1] = (float)adv; o[2] = (float)(l01 * (double)(float)w01m); o[3] = (float)ltot; o[4] = (float)ltv;
                    o[5] = (float)closs; o[6] = (float)w; o[7] = (float)cl;
                    if (hp.gan_on && hp.matching) hist_gan[(long)g * R + (hp.head_gan + hp.hist_size) % R] = adv32;
                    if (hp.council_on && hp.matching)
                        hist_council[(long)g * R + (hp.head_council + hp.hist_size) % R] = (double)(float)cl;
                    if (fm && hp.w01 != 0.0) hp.hist_focus01[(long)g * R + (hp.head_focus01 + hp.hist_size) % R] = l01_32;
                    if (fm && hp.wtot != 0.0) hp.hist_focus[(long)g * R + (hp.head_focus + hp.hist_size) % R] = ltot_app;
                    if (hp.focus_w) { hp.focus_w[g * 2] = (float)w01m; hp.focus_w[g * 2 + 1] = (float)wtm; }
                }
            }
        }
    }
    __syncthreads();
    // ---- gradients ------------------------------------------------------------------------------------------------
    if ((int)blockIdx.x < map_blocks) {
        // council-D patch maps: d out = cdis[g] * 2 / (n * world) * (out - 1), one block per (map, member)
        const int m = blockIdx.x / G, g = blockIdx.x - m * G;
        const int n = d.cl_n[m];
        const float coef = sc[g].cdis * (2.0f / ((float)n * (float)hp.world));
        const float* p = d.cl_out[m] + (long)g * n;
        float* q = d.cl_dout[m] + (long)g * n;
        for (int i = threadIdx.x; i < n; i += blockDim.x) q[i] = coef * (__ldg(p + i) - 1.0f);
        return;
    }
    if (!d_mask) return;
    const int H = d.H, W = d.W;
    const long npix = (long)d.B * H * W, total_px = npix * G;
    const float center = d.center, eps = d.eps;
    const long stride = (long)(gridDim.x - map_blocks) * blockDim.x;
    for (long i = (long)(blockIdx.x - map_blocks) * blockDim.x + threadIdx.x; i < total_px; i += stride) {
        const int g = (int)(i / npix);
        const long px = i - (long)g * npix;
        const int w = (int)(px % W);
        const int h = (int)((px / W) % H);
        const float c01 = sc[g].c01, cs = sc[g].csum, ctv = sc[g].ctv;
        const float* mp = d.mask + i * 4;
        float4 mk = ld4(mp);
        float mm[3] = {mk.x, mk.y, mk.z}, o[3];
#pragma unroll
        for (int c = 0; c < 3; c++) {
            float df = mm[c] - center;
            float den = fabsf(df) + eps;
            o[c] = cs - c01 * sgnf(df) / (den * den);
        }
        if (ctv != 0.f) {
            float tv[3] = {0.f, 0.f, 0.f};
            if (h + 1 < H) { float4 q = ld4(mp + (long)W * 4); tv[0] -= sgnf(q.x - mk.x); tv[1] -= sgnf(q.y - mk.y); tv[2] -= sgnf(q.z - mk.z); }
            if (h > 0)     { float4 q = ld4(mp - (long)W * 4); tv[0] += sgnf(mk.x - q.x); tv[1] += sgnf(mk.y - q.y); tv[2] += sgnf(mk.z - q.z); }
            if (w + 1 < W) { float4 q = ld4(mp + 4);           tv[0] -= sgnf(q.x - mk.x); tv[1] -= sgnf(q.y - mk.y); tv[2] -= sgnf(q.z - mk.z); }
            if (w > 0)     { float4 q = ld4(mp - 4);           tv[0] += sgnf(mk.x - q.x); tv[1] += sgnf(mk.y - q.y); tv[2] += sgnf(mk.z - q.z); }
#pragma unroll
            for (int c = 0; c < 3; c++) o[c] += ctv * tv[c];
        }
        reinterpret_cast<float4*>(d_mask)[i] = make_float4(o[0], o[1], o[2], 0.f);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// gen_update, abs_beginning_end: recon_criterion_v2_color(x_fake, x) (trainer_council.py:210-215, 477-495), d = x_fake - x
// over the 3 live lanes; L1 = mean |d|, L2 = mean d^2, the loss is L1 if L1 > L2 else L2
// ---------------------------------------------------------------------------------------------------------------
// pass 1: block (chunk, g) sums |d| and d^2 over GL_PIX pixels in float, the last block adds the chunks in double (the
// convention of the focus sums).  part: float [nchunks][G][2].
__global__ void __launch_bounds__(256) abs_be_fwd_kernel(const float* __restrict__ x_fake, const float* __restrict__ x, float* __restrict__ sums,
                                                         float* __restrict__ part, unsigned int* __restrict__ counter, int G, long npix,
                                                         int nchunks) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sm[2 * 32];
    const int g = blockIdx.x % G, chunk = blockIdx.x / G;
    const long p0 = (long)chunk * GL_PIX, p1 = min(npix, p0 + GL_PIX);
    const float* xf = x_fake + (long)g * npix * 4;
    float v[2] = {0.f, 0.f};
    for (long px = p0 + threadIdx.x; px < p1; px += blockDim.x) {
        const float4 a = ld4(xf + px * 4), b = ld4(x + px * 4);
        const float d0 = a.x - b.x, d1 = a.y - b.y, d2 = a.z - b.z;
        v[0] += fabsf(d0) + fabsf(d1) + fabsf(d2);
        v[1] += d0 * d0 + d1 * d1 + d2 * d2;
    }
    block_sum<2>(v, sm);
    if (threadIdx.x == 0) {
        float* o = part + ((long)chunk * G + g) * 2;
        o[0] = v[0]; o[1] = v[1];
    }
    if (!last_block_done(counter, gridDim.x)) return;
    const int t = threadIdx.x;  // sums[g][k] = sum over chunks of part[c][g][k], k = 0 (|d|), 1 (d^2)
    if (t < G * 2) {
        const volatile float* vp = part;
        double s = 0.0;
        for (int c = 0; c < nchunks; c++) s += (double)vp[(long)c * G * 2 + t];
        sums[t] = (float)s;
    }
    if (t == 0) *counter = 0u;
}

struct AbsBeWeights { double w[CG_LOSS_MAX_G]; };  // per member; 0: no contribution (the member's gate is closed)

// pass 2 (sums summed over ranks): every block derives the branch and the gradient coefficient of each member; block 0 publishes
// the unweighted loss and adds w * loss to the double accumulator of the direction totals (the one cg_gen_loss_bwd keeps in the
// same workspace); then a grid-stride pass adds the gradient to d_x: w/numel * sign(d) (L1; sign(0) = 0) or w/numel * 2d (L2).
__global__ void __launch_bounds__(256) abs_be_bwd_kernel(const float* __restrict__ x_fake, const float* __restrict__ x, const float* __restrict__ sums,
                                                         double numel, const AbsBeWeights wt, int G, long npix, float* __restrict__ total,
                                                         double* __restrict__ total64, float* __restrict__ pub, float* __restrict__ d_x) {
    pdl_trigger();
    pdl_wait();
    __shared__ float s_coef[CG_LOSS_MAX_G];
    __shared__ int s_l1[CG_LOSS_MAX_G];
    if (threadIdx.x < G) {
        const int g = threadIdx.x;
        const double l1 = (double)sums[2 * g] / numel, l2 = (double)sums[2 * g + 1] / numel;
        const bool use_l1 = l1 > l2;  // a tie picks L2
        const double val = use_l1 ? l1 : l2, w = wt.w[g];
        s_l1[g] = use_l1;
        s_coef[g] = (float)((use_l1 ? 1.0 : 2.0) * w / numel);
        if (blockIdx.x == 0) {
            pub[g] = (float)val;
            if (w != 0.0) {
                const double t64 = total64[g] + w * val;
                total64[g] = t64;
                total[g] = (float)t64;
            }
        }
    }
    __syncthreads();
    const long total_px = npix * G, stride = (long)gridDim.x * blockDim.x;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total_px; i += stride) {
        const int g = (int)(i / npix);
        const float c = s_coef[g];
        if (c == 0.f) continue;
        const float4 a = ld4(x_fake + i * 4), b = ld4(x + (i - (long)g * npix) * 4);
        const float d0 = a.x - b.x, d1 = a.y - b.y, d2 = a.z - b.z;
        float4 o = reinterpret_cast<const float4*>(d_x)[i];
        if (s_l1[g]) {
            o.x += c * sgnf(d0); o.y += c * sgnf(d1); o.z += c * sgnf(d2);
        } else {
            o.x += c * d0; o.y += c * d1; o.z += c * d2;
        }
        reinterpret_cast<float4*>(d_x)[i] = o;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// gen_update, council abs loss (council_abs_w, trainer_council.py:224-228, 595-619): member g's translation against the detached
// translation of its peer p[g], mean |x_g - x_p| over the 3 live lanes (colour) or mean |sum_c x_g - sum_c x_p| (gray scale)
// ---------------------------------------------------------------------------------------------------------------
struct CouncilPeers { int p[CG_LOSS_MAX_G]; };  // host-drawn peers, passed by value

// pr.p[g] without a dynamic index into the parameter struct (which would copy it to the stack)
__device__ __forceinline__ int peer_of(const CouncilPeers& pr, int g) {
    int p = 0;
#pragma unroll
    for (int k = 0; k < CG_LOSS_MAX_G; k++) p = k == g ? pr.p[k] : p;
    return p;
}

// |x_g - x_p| of one pixel (colour: 3 lanes; gray: the channel sums, as torch.sum(x, 1) - torch.sum(y, 1))
__device__ __forceinline__ float council_abs_pix(const float4 a, const float4 b, int gray) {
    return gray ? fabsf((a.x + a.y + a.z) - (b.x + b.y + b.z)) : fabsf(a.x - b.x) + fabsf(a.y - b.y) + fabsf(a.z - b.z);
}

// pass 1: block (chunk, g) sums over GL_PIX pixels in float, the last block adds the chunks in double, in chunk order (the convention
// of abs_be_fwd_kernel).  part: float [nchunks][G].
__global__ void __launch_bounds__(256) council_abs_fwd_kernel(const float* __restrict__ x_fake, const CouncilPeers pr, int gray,
                                                              float* __restrict__ sums, float* __restrict__ part,
                                                              unsigned int* __restrict__ counter, int G, long npix, int nchunks) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sm[32];
    const int g = blockIdx.x % G, chunk = blockIdx.x / G;
    const long p0 = (long)chunk * GL_PIX, p1 = min(npix, p0 + GL_PIX);
    const float* xg = x_fake + (long)g * npix * 4;
    const float* xp = x_fake + (long)peer_of(pr, g) * npix * 4;
    float v[1] = {0.f};
    for (long px = p0 + threadIdx.x; px < p1; px += blockDim.x) v[0] += council_abs_pix(ld4(xg + px * 4), ld4(xp + px * 4), gray);
    block_sum<1>(v, sm);
    if (threadIdx.x == 0) part[(long)chunk * G + g] = v[0];
    if (!last_block_done(counter, gridDim.x)) return;
    const int t = threadIdx.x;
    if (t < G) {
        const volatile float* vp = part;
        double s = 0.0;
        for (int c = 0; c < nchunks; c++) s += (double)vp[(long)c * G + t];
        sums[t] = (float)s;
    }
    if (t == 0) *counter = 0u;
}

// pass 2 (sums summed over ranks, numel of the GLOBAL minibatch): block 0 publishes the weighted term pub[g] = w * sums[g] / numel and
// adds it to the double accumulator of the direction totals; a grid-stride pass adds w / numel * sign(d) to d_x on lanes 0..2 (gray:
// the sign of the channel-sum difference on all three), sign(0) = 0.  The peer's image takes no gradient.
__global__ void __launch_bounds__(256) council_abs_bwd_kernel(const float* __restrict__ x_fake, const CouncilPeers pr, int gray,
                                                              const float* __restrict__ sums, double numel, double w, int G, long npix,
                                                              float* __restrict__ total, double* __restrict__ total64,
                                                              float* __restrict__ pub, float* __restrict__ d_x) {
    pdl_trigger();
    pdl_wait();
    __shared__ long s_off[CG_LOSS_MAX_G];  // pixel offset of member g's peer
    if ((int)threadIdx.x < G) {
        const int g = threadIdx.x;
        s_off[g] = (long)(peer_of(pr, g) - g) * npix;
        if (blockIdx.x == 0) {
            const double term = w * ((double)sums[g] / numel);
            pub[g] = (float)term;
            const double t64 = total64[g] + term;
            total64[g] = t64;
            total[g] = (float)t64;
        }
    }
    __syncthreads();
    const float c = (float)(w / numel);
    const long total_px = npix * G, stride = (long)gridDim.x * blockDim.x;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total_px; i += stride) {
        const int g = (int)(i / npix);
        const float4 a = ld4(x_fake + i * 4), b = ld4(x_fake + (i + s_off[g]) * 4);
        float4 o = reinterpret_cast<const float4*>(d_x)[i];
        if (gray) {
            const float s = c * sgnf((a.x + a.y + a.z) - (b.x + b.y + b.z));
            o.x += s; o.y += s; o.z += s;
        } else {
            o.x += c * sgnf(a.x - b.x); o.y += c * sgnf(a.y - b.y); o.z += c * sgnf(a.z - b.z);
        }
        reinterpret_cast<float4*>(d_x)[i] = o;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// gen_update, latent reconstruction (recon_c_w / recon_s_w, trainer_council.py:359-369, 460-469): recon_criterion = mean |a - b|
// of a re-encoded content / style code a against its target b
// ---------------------------------------------------------------------------------------------------------------
constexpr int L1_THREADS = 256, L1_MAX_BLOCKS = 256;  // blocks per member

// block (j, g) walks member g's n elements with stride nb * 256 (fixed for a shape: the float partial of a block and therefore the
// sum are deterministic); the last block adds each member's partials in double, in block order.  The gradient does not depend on
// the loss value: da (+)= coef * sign(a - b), db (+)= -coef * sign(a - b) in the same pass (sign(0) = 0).
template <bool VEC>
__global__ void __launch_bounds__(L1_THREADS) latent_l1_kernel(const float* __restrict__ a, const float* __restrict__ b, int b_shared, long n,
                                                               float* __restrict__ da, float* __restrict__ db, float coef, int accumulate,
                                                               float* __restrict__ sums, float* __restrict__ part,
                                                               unsigned int* __restrict__ counter, int G, int nb) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sm[32];
    const int g = blockIdx.x / nb, j = blockIdx.x - g * nb;
    const long base = (long)g * n, bbase = b_shared ? 0 : base;
    float v[1] = {0.f};
    if (VEC) {
        const long n4 = n / 4;
        const float4* a4 = reinterpret_cast<const float4*>(a + base);
        const float4* b4 = reinterpret_cast<const float4*>(b + bbase);
        float4* da4 = da ? reinterpret_cast<float4*>(da + base) : nullptr;
        float4* db4 = db ? reinterpret_cast<float4*>(db + base) : nullptr;
        for (long i = (long)j * L1_THREADS + threadIdx.x; i < n4; i += (long)nb * L1_THREADS) {
            const float4 x = __ldg(a4 + i), y = __ldg(b4 + i);
            const float d0 = x.x - y.x, d1 = x.y - y.y, d2 = x.z - y.z, d3 = x.w - y.w;
            v[0] += fabsf(d0) + fabsf(d1) + fabsf(d2) + fabsf(d3);
            const float4 gr = make_float4(coef * sgnf(d0), coef * sgnf(d1), coef * sgnf(d2), coef * sgnf(d3));
            if (da4) {
                float4 o = accumulate ? da4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
                o.x += gr.x; o.y += gr.y; o.z += gr.z; o.w += gr.w;
                da4[i] = o;
            }
            if (db4) {
                float4 o = accumulate ? db4[i] : make_float4(0.f, 0.f, 0.f, 0.f);
                o.x -= gr.x; o.y -= gr.y; o.z -= gr.z; o.w -= gr.w;
                db4[i] = o;
            }
        }
    } else {
        for (long i = (long)j * L1_THREADS + threadIdx.x; i < n; i += (long)nb * L1_THREADS) {
            const float d = __ldg(a + base + i) - __ldg(b + bbase + i);
            v[0] += fabsf(d);
            const float gr = coef * sgnf(d);
            if (da) da[base + i] = (accumulate ? da[base + i] : 0.f) + gr;
            if (db) db[base + i] = (accumulate ? db[base + i] : 0.f) - gr;
        }
    }
    block_sum<1>(v, sm);
    if (threadIdx.x == 0) part[blockIdx.x] = v[0];
    if (!last_block_done(counter, gridDim.x)) return;
    if (threadIdx.x < G) {
        const volatile float* vp = part + (long)threadIdx.x * nb;
        double s = 0.0;
        for (int k = 0; k < nb; k++) s += (double)vp[k];
        sums[threadIdx.x] = (float)s;
    }
    if (threadIdx.x == 0) *counter = 0u;
}

// ---------------------------------------------------------------------------------------------------------------
// gen_update, image reconstruction (recon_x_w, trainer_council.py:339-345, 455-459): x_recon = the attention-mask composite of the
// other direction's decoder head over the source image x; recon_criterion = mean |x_recon - x| over the 3 live lanes.  x_recon
// feeds only this loss, so it is never written: pass 1 reduces the sums, the backward recomputes the composite (mask_head.cuh).
// ---------------------------------------------------------------------------------------------------------------
// pass 1: block (chunk, g) sums |x_recon - x| over GL_PIX pixels in float, the last block adds the chunks in double, in chunk order
// (the convention of abs_be_fwd_kernel).  h [G][npix][12] (tanh output of the last head layer), x [npix][4] shared; part: float
// [nchunks][G].
__global__ void __launch_bounds__(256) recon_head_fwd_kernel(const float* __restrict__ h, const float* __restrict__ x, float* __restrict__ sums,
                                                             float* __restrict__ part, unsigned int* __restrict__ counter, int G, long npix,
                                                             int nchunks) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sm[32];
    const int g = blockIdx.x % G, chunk = blockIdx.x / G;
    const long p0 = (long)chunk * GL_PIX, p1 = min(npix, p0 + GL_PIX);
    const float* hg = h + (long)g * npix * 12;
    float v[1] = {0.f};
    for (long px = p0 + threadIdx.x; px < p1; px += blockDim.x) {
        MaskHeadPix p;
        mask_composite(hg + px * 12, x + px * 4, p);
        v[0] += fabsf(p.im[3][0] - p.im[0][0]) + fabsf(p.im[3][1] - p.im[0][1]) + fabsf(p.im[3][2] - p.im[0][2]);
    }
    block_sum<1>(v, sm);
    if (threadIdx.x == 0) part[(long)chunk * G + g] = v[0];
    if (!last_block_done(counter, gridDim.x)) return;
    const int t = threadIdx.x;
    if (t < G) {
        const volatile float* vp = part;
        double s = 0.0;
        for (int c = 0; c < nchunks; c++) s += (double)vp[(long)c * G + t];
        sums[t] = (float)s;
    }
    if (t == 0) *counter = 0u;
}

// backward: d(x_recon) = coef * sign(x_recon - x) (sign(0) = 0; coef = recon_x_w / numel of the GLOBAL minibatch) through the
// composite and the head's tanh, as mask_head_bwd_kernel with d_mask = 0: dh_pre [G][npix][12]
__global__ void __launch_bounds__(256) recon_head_bwd_kernel(const float* __restrict__ h, const float* __restrict__ x, float coef,
                                                             float* __restrict__ dh_pre, long total, long npix) {
    pdl_trigger();
    pdl_wait();
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    MaskHeadPix p;
    mask_composite(h + i * 12, x + (i % npix) * 4, p);
    float dim[3];
#pragma unroll
    for (int ch = 0; ch < 3; ch++) dim[ch] = coef * sgnf(p.im[3][ch] - p.im[0][ch]);
    const float dm[3] = {0.f, 0.f, 0.f};
    float out[12];
    mask_head_grad(p, dim, dm, out);
    store12(dh_pre + i * 12, out);
}

// ---------------------------------------------------------------------------------------------------------------
// gen_update, perceptual loss (vgg_w, trainer_council.py:531-538, 636-641): mean((IN(f_img) - IN(f_tgt))^2) of relu5_3 features,
// IN = nn.InstanceNorm2d(512, affine=False) (:121), and its gradient w.r.t. conv5_3's pre-activation
// ---------------------------------------------------------------------------------------------------------------
constexpr int VL_CH = 32, VL_PY = 8;  // channels x pixel lanes of a 256-thread block

// block (r, chunk) owns channels [32 chunk, 32 chunk + 32) of image row r and pairs it with target row t(r) = (r / per_dir) * B + r % B.
// Pass 1 over the pixels: z = (f - mean) * rstd of both, d = z_img - z_tgt; the float partial sum d^2 of the block, and per channel
// mean(g) and mean(g z_img) of g = 2 coef d.  Pass 2: d_pre = rstd (g - mean(g) - z_img mean(g z_img)) (the instance-norm backward,
// statistics included) times relu5_3's mask f > 0.  The last block adds the partials of each term k (rows [k B, k B + B), the
// blocks of a row in chunk order) in double: sums[k].
__global__ void __launch_bounds__(256) vgg_loss_kernel(const float* __restrict__ fi, const float* __restrict__ mi, const float* __restrict__ ri,
                                                       const float* __restrict__ ft, const float* __restrict__ mt, const float* __restrict__ rt,
                                                       float coef, float* __restrict__ d_pre, float* __restrict__ sums,
                                                       float* __restrict__ part, unsigned int* __restrict__ counter, int B, int per_dir,
                                                       int HW, int C, int nterm) {
    pdl_trigger();
    pdl_wait();
    __shared__ float sm[32];
    __shared__ float red[2][VL_PY][VL_CH];
    const int nchunk = C / VL_CH;
    const int r = blockIdx.x / nchunk, chunk = blockIdx.x - r * nchunk;
    const int tr = (r / per_dir) * B + r % B;
    const int lane = threadIdx.x & 31, py = threadIdx.x >> 5;
    const int c = chunk * VL_CH + lane;
    const float m_i = __ldg(mi + (long)r * C + c), r_i = __ldg(ri + (long)r * C + c);
    const float m_t = __ldg(mt + (long)tr * C + c), r_t = __ldg(rt + (long)tr * C + c);
    const float* fr = fi + (long)r * HW * C + c;
    const float* ftr = ft + (long)tr * HW * C + c;
    const float two_coef = 2.f * coef;
    float v[1] = {0.f};
    float sg = 0.f, sgz = 0.f;
    for (int p = py; p < HW; p += VL_PY) {
        const float zi = (__ldg(fr + (long)p * C) - m_i) * r_i;
        const float d = zi - (__ldg(ftr + (long)p * C) - m_t) * r_t;
        v[0] += d * d;
        const float g = two_coef * d;
        sg += g;
        sgz += g * zi;
    }
    red[0][py][lane] = sg;
    red[1][py][lane] = sgz;
    block_sum<1>(v, sm);  // its barriers also publish red
    float mg = 0.f, mgz = 0.f;
#pragma unroll
    for (int k = 0; k < VL_PY; k++) {
        mg += red[0][k][lane];
        mgz += red[1][k][lane];
    }
    mg /= (float)HW;
    mgz /= (float)HW;
    float* dr = d_pre + (long)r * HW * C + c;
    for (int p = py; p < HW; p += VL_PY) {
        const float f = __ldg(fr + (long)p * C);
        const float zi = (f - m_i) * r_i;
        const float g = two_coef * (zi - (__ldg(ftr + (long)p * C) - m_t) * r_t);
        dr[(long)p * C] = f > 0.f ? r_i * (g - mg - zi * mgz) : 0.f;
    }
    if (threadIdx.x == 0) part[blockIdx.x] = v[0];
    if (!last_block_done(counter, gridDim.x)) return;
    const int t = threadIdx.x;
    if (t < nterm) {
        const volatile float* vp = part + (long)t * B * nchunk;
        double s = 0.0;
        for (int k = 0; k < B * nchunk; k++) s += (double)vp[k];
        sums[t] = (float)s;
    }
    if (t == 0) *counter = 0u;
}

struct ReconTerms { double numel[CG_RECON_MAX_TERMS], w[CG_RECON_MAX_TERMS]; };

// after the all-reduce: pub[k][g] = sums[k][g] / numel[k]; total[g] += sum_k w[k] * pub[k][g] through the double accumulator of
// the direction totals (the one cg_gen_loss_bwd keeps in the same workspace)
__global__ void recon_finalize_kernel(const float* __restrict__ sums, const ReconTerms t, int nterm, int G, float* __restrict__ total,
                                      double* __restrict__ total64, float* __restrict__ pub) {
    pdl_trigger();
    pdl_wait();
    const int g = threadIdx.x;
    if (g >= G) return;
    double t64 = total64[g];
    bool any = false;
    for (int k = 0; k < nterm; k++) {
        const double val = (double)sums[k * G + g] / t.numel[k];
        pub[k * G + g] = (float)val;
        if (t.w[k] != 0.0) {
            t64 += t.w[k] * val;
            any = true;
        }
    }
    if (any) {
        total64[g] = t64;
        total[g] = (float)t64;
    }
}

}  // namespace cg

using namespace cg;
#define ST ((cudaStream_t)stream)

extern "C" size_t cg_loss_workspace_bytes(int G, int B, int H, int W) {
    long npix = (long)B * H * W;
    size_t nchunks = (size_t)cdiv(npix > 0 ? npix : 1, GL_PIX);
    // maps partials (<= 4 maps x G x 8 segments) + focus partials + ticket + the double accumulators of pass 2
    return 16 + (size_t)CG_LOSS_MAX_MAPS * CG_LOSS_MAX_G * CG_LOSS_MAX_SEG * 4 + nchunks * (size_t)G * 16 + CG_LOSS_MAX_G * 8;
}

// workspace layout (all three calls): [0,16) ticket counter (must be zero on entry; left zero), then double total64[MAX_G],
// then float partials
static inline unsigned int* ws_counter(void* ws) { return (unsigned int*)ws; }
static inline double* ws_total64(void* ws) { return (double*)((char*)ws + 16); }
static inline float* ws_part(void* ws) { return (float*)((char*)ws + 16 + CG_LOSS_MAX_G * 8); }

extern "C" int cg_lsgan_fused(const cg_lsgan_desc* d, float* loss_total, int accumulate, float* loss_plain, void* ws,
                              size_t ws_bytes, void* stream) {
    CG_REQUIRE(d && d->nmaps >= 1 && d->nmaps <= CG_LOSS_MAX_MAPS && d->G >= 1 && d->G <= CG_LOSS_MAX_G && d->nseg >= 1 &&
               d->nseg <= CG_LOSS_MAX_SEG, "lsgan_fused: nmaps=%d G=%d nseg=%d out of range", d ? d->nmaps : -1, d ? d->G : -1,
               d ? d->nseg : -1);
    size_t need = 16 + CG_LOSS_MAX_G * 8 + (size_t)d->nmaps * d->G * d->nseg * 4;
    if (need > ws_bytes) {
        set_error("lsgan_fused: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    for (int m = 0; m < d->nmaps; m++) CG_REQUIRE(d->out[m] && d->n_per_seg[m] > 0, "lsgan_fused: map %d is empty", m);
    int blocks = d->nmaps * d->G * d->nseg;
    launch_k(lsgan_fused_kernel, blocks, 256, 0, ST, *d, loss_total, accumulate, loss_plain, ws_part(ws), ws_counter(ws));
    return check_launch("lsgan_fused");
}

static int check_gen_desc(const cg_gen_loss_desc* d, const char* who) {
    CG_REQUIRE(d && d->G >= 1 && d->G <= CG_LOSS_MAX_G && d->n_adv >= 0 && d->n_adv <= 2 && d->n_cl >= 0 && d->n_cl <= 2,
               "%s: G / map counts out of range", who);
    CG_REQUIRE(d->G * 6 <= 256, "%s: G too large", who);
    return CG_OK;
}

extern "C" int cg_gen_loss_fwd(const cg_gen_loss_desc* d, float* scal, void* ws, size_t ws_bytes, void* stream) {
    if (int rc = check_gen_desc(d, "gen_loss_fwd")) return rc;
    long npix = (long)d->B * d->H * d->W;
    int nchunks = d->mask ? cdiv(npix, GL_PIX) : 0;
    int nmaps = d->n_adv + d->n_cl;
    size_t need = 16 + CG_LOSS_MAX_G * 8 + ((size_t)nmaps * d->G + (size_t)nchunks * d->G * 4) * 4;
    if (need > ws_bytes) {
        set_error("gen_loss_fwd: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    int blocks = nmaps * d->G + nchunks * d->G;
    if (blocks == 0) {  // nothing to reduce: all six scalars are zero
        cudaError_t e = cudaMemsetAsync(scal, 0, (size_t)d->G * 6 * 4, ST);
        if (e != cudaSuccess) {
            set_error("gen_loss_fwd: %s", cudaGetErrorString(e));
            return CG_ERR_CUDA;
        }
        return CG_OK;
    }
    float* part_map = ws_part(ws);
    float* part_focus = part_map + (size_t)nmaps * d->G;
    launch_k(gen_loss_fwd_kernel, blocks, 256, 0, ST, *d, scal, part_map, part_focus, ws_counter(ws), nchunks);
    return check_launch("gen_loss_fwd");
}

extern "C" int cg_gen_loss_bwd(const cg_gen_loss_desc* d, const cg_gen_loss_hp* hp, const float* scal, double* hist_gan,
                               double* hist_council, float* total, int accumulate, float* pub, float* d_mask, void* ws,
                               size_t ws_bytes, void* stream) {
    if (int rc = check_gen_desc(d, "gen_loss_bwd")) return rc;
    CG_REQUIRE(hp && hp->world >= 1 && hp->hist_size >= 1 && hp->numel > 0, "gen_loss_bwd: bad hyper-parameters");
    CG_REQUIRE(ws_bytes >= 16 + CG_LOSS_MAX_G * 8, "gen_loss_bwd: workspace too small");
    CG_REQUIRE(!d_mask || d->mask, "gen_loss_bwd: d_mask without mask");
    if (hp->focus_matching && hp->focus_on) {
        CG_REQUIRE((hp->w01 == 0.0 || hp->hist_focus01) && (hp->wtot == 0.0 || hp->hist_focus),
                   "gen_loss_bwd: focus matching without its history rings");
        CG_REQUIRE(hp->head_focus >= 0 && hp->head_focus <= hp->hist_size && hp->head_focus01 >= 0 && hp->head_focus01 <= hp->hist_size,
                   "gen_loss_bwd: focus history heads out of range");
    }
    for (int m = 0; m < d->n_cl; m++) CG_REQUIRE(d->cl_dout[m] && d->cl_out[m], "gen_loss_bwd: council map %d without buffers", m);
    int map_blocks = d->n_cl * d->G;
    long total_px = d_mask ? (long)d->G * d->B * d->H * d->W : 0;
    int px_blocks = d_mask ? cdiv(total_px, 256) : 0;
    const int px_cap = 8 * (tc_sm_count() > 0 ? tc_sm_count() : 1);  // grid-stride: each block pays the finalise prologue once
    if (px_blocks > px_cap) px_blocks = px_cap;
    int blocks = map_blocks + px_blocks;
    if (blocks == 0) blocks = 1;  // the finalise / publish step always runs
    launch_k(gen_loss_bwd_kernel, blocks, 256, 0, ST, *d, *hp, scal, hist_gan, hist_council, total, ws_total64(ws), accumulate, pub, d_mask,
                                                map_blocks);
    return check_launch("gen_loss_bwd");
}

extern "C" int cg_abs_beginning_end_fwd(const float* x_fake, const float* x, float* sums, int G, int B, int H, int W, void* ws,
                                        size_t ws_bytes, void* stream) {
    CG_REQUIRE(x_fake && x && sums && G >= 1 && G <= CG_LOSS_MAX_G && B >= 1 && H >= 1 && W >= 1,
               "abs_beginning_end_fwd: G=%d B=%d H=%d W=%d out of range", G, B, H, W);
    const long npix = (long)B * H * W;
    const int nchunks = cdiv(npix, GL_PIX);
    size_t need = 16 + CG_LOSS_MAX_G * 8 + (size_t)nchunks * G * 2 * 4;
    if (need > ws_bytes) {
        set_error("abs_beginning_end_fwd: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    launch_k(abs_be_fwd_kernel, nchunks * G, 256, 0, ST, x_fake, x, sums, ws_part(ws), ws_counter(ws), G, npix, nchunks);
    return check_launch("abs_beginning_end_fwd");
}

extern "C" int cg_abs_beginning_end_bwd(const float* x_fake, const float* x, const float* sums, double numel, const double* host_weight,
                                        float* total, float* pub, float* d_x, int G, int B, int H, int W, void* ws, size_t ws_bytes,
                                        void* stream) {
    CG_REQUIRE(x_fake && x && sums && host_weight && total && pub && d_x && G >= 1 && G <= CG_LOSS_MAX_G && B >= 1 && H >= 1 && W >= 1,
               "abs_beginning_end_bwd: G=%d B=%d H=%d W=%d out of range", G, B, H, W);
    CG_REQUIRE(numel > 0, "abs_beginning_end_bwd: numel must be positive");
    CG_REQUIRE(ws_bytes >= 16 + CG_LOSS_MAX_G * 8, "abs_beginning_end_bwd: workspace too small");
    AbsBeWeights wt = {};
    for (int g = 0; g < G; g++) wt.w[g] = host_weight[g];
    const long npix = (long)B * H * W;
    int blocks = cdiv(npix * G, 256);
    const int cap = 8 * (tc_sm_count() > 0 ? tc_sm_count() : 1);
    if (blocks > cap) blocks = cap;
    launch_k(abs_be_bwd_kernel, blocks, 256, 0, ST, x_fake, x, sums, numel, wt, G, npix, total, ws_total64(ws), pub, d_x);
    return check_launch("abs_beginning_end_bwd");
}

static int council_peers(const int32_t* host_peer, int G, CouncilPeers& pr, const char* who) {
    CG_REQUIRE(host_peer && G >= 1 && G <= CG_LOSS_MAX_G, "%s: G=%d out of range", who, G);
    for (int g = 0; g < G; g++) {
        CG_REQUIRE(host_peer[g] >= 0 && host_peer[g] < G && host_peer[g] != g, "%s: peer %d of member %d is not another member", who,
                   host_peer[g], g);
        pr.p[g] = host_peer[g];
    }
    return CG_OK;
}

extern "C" int cg_council_abs_fwd(const float* x_fake, const int32_t* host_peer, int gray, float* sums, int G, int B, int H, int W,
                                  void* ws, size_t ws_bytes, void* stream) {
    CouncilPeers pr = {};
    if (int rc = council_peers(host_peer, G, pr, "council_abs_fwd")) return rc;
    CG_REQUIRE(x_fake && sums && B >= 1 && H >= 1 && W >= 1, "council_abs_fwd: B=%d H=%d W=%d out of range", B, H, W);
    const long npix = (long)B * H * W;
    const int nchunks = cdiv(npix, GL_PIX);
    size_t need = 16 + CG_LOSS_MAX_G * 8 + (size_t)nchunks * G * 4;
    if (need > ws_bytes) {
        set_error("council_abs_fwd: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    launch_k(council_abs_fwd_kernel, nchunks * G, 256, 0, ST, x_fake, pr, gray, sums, ws_part(ws), ws_counter(ws), G, npix, nchunks);
    return check_launch("council_abs_fwd");
}

extern "C" int cg_council_abs_bwd(const float* x_fake, const int32_t* host_peer, int gray, const float* sums, double numel, double w,
                                  float* total, float* pub, float* d_x, int G, int B, int H, int W, void* ws, size_t ws_bytes,
                                  void* stream) {
    CouncilPeers pr = {};
    if (int rc = council_peers(host_peer, G, pr, "council_abs_bwd")) return rc;
    CG_REQUIRE(x_fake && sums && total && pub && d_x && B >= 1 && H >= 1 && W >= 1, "council_abs_bwd: B=%d H=%d W=%d out of range", B,
               H, W);
    CG_REQUIRE(numel > 0, "council_abs_bwd: numel must be positive");
    CG_REQUIRE(ws_bytes >= 16 + CG_LOSS_MAX_G * 8, "council_abs_bwd: workspace too small");
    const long npix = (long)B * H * W;
    int blocks = cdiv(npix * G, 256);
    const int cap = 8 * (tc_sm_count() > 0 ? tc_sm_count() : 1);
    if (blocks > cap) blocks = cap;
    launch_k(council_abs_bwd_kernel, blocks, 256, 0, ST, x_fake, pr, gray, sums, numel, w, G, npix, total, ws_total64(ws), pub, d_x);
    return check_launch("council_abs_bwd");
}

static int latent_l1_blocks(long n) {
    const long units = n % 4 == 0 ? n / 4 : n;
    int nb = cdiv(units, (long)L1_THREADS * 8);
    return nb < 1 ? 1 : (nb > L1_MAX_BLOCKS ? L1_MAX_BLOCKS : nb);
}

extern "C" int cg_latent_l1(const float* a, const float* b, int b_shared, float* da, float* db, float coef, int accumulate, float* sums,
                            int G, long n, void* ws, size_t ws_bytes, void* stream) {
    CG_REQUIRE(a && b && sums && G >= 1 && G <= CG_LOSS_MAX_G && n >= 1, "latent_l1: G=%d n=%ld out of range", G, n);
    CG_REQUIRE(!(db && b_shared), "latent_l1: a target shared by all members cannot take a gradient");
    const int nb = latent_l1_blocks(n);
    size_t need = 16 + CG_LOSS_MAX_G * 8 + (size_t)G * nb * 4;
    if (need > ws_bytes) {
        set_error("latent_l1: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    if (n % 4 == 0)
        launch_k(latent_l1_kernel<true>, G * nb, L1_THREADS, 0, ST, a, b, b_shared, n, da, db, coef, accumulate, sums, ws_part(ws),
                 ws_counter(ws), G, nb);
    else
        launch_k(latent_l1_kernel<false>, G * nb, L1_THREADS, 0, ST, a, b, b_shared, n, da, db, coef, accumulate, sums, ws_part(ws),
                 ws_counter(ws), G, nb);
    return check_launch("latent_l1");
}

extern "C" int cg_recon_finalize(const float* sums, const double* host_numel, const double* host_weight, int nterm, int G, float* total,
                                 float* pub, void* ws, size_t ws_bytes, void* stream) {
    CG_REQUIRE(sums && host_numel && host_weight && total && pub && nterm >= 1 && nterm <= CG_RECON_MAX_TERMS && G >= 1 &&
               G <= CG_LOSS_MAX_G, "recon_finalize: nterm=%d G=%d out of range", nterm, G);
    CG_REQUIRE(ws_bytes >= 16 + CG_LOSS_MAX_G * 8, "recon_finalize: workspace too small");
    ReconTerms t = {};
    for (int k = 0; k < nterm; k++) {
        CG_REQUIRE(host_numel[k] > 0, "recon_finalize: numel must be positive");
        t.numel[k] = host_numel[k];
        t.w[k] = host_weight[k];
    }
    launch_k(recon_finalize_kernel, 1, 32, 0, ST, sums, t, nterm, G, total, ws_total64(ws), pub);
    return check_launch("recon_finalize");
}

extern "C" int cg_recon_head_fwd(const float* h, const float* x, float* sums, int G, int B, int HW, void* ws, size_t ws_bytes, void* stream) {
    CG_REQUIRE(h && x && sums && G >= 1 && G <= CG_LOSS_MAX_G && B >= 1 && HW >= 1, "recon_head_fwd: G=%d B=%d HW=%d out of range", G, B,
               HW);
    const long npix = (long)B * HW;
    const int nchunks = cdiv(npix, GL_PIX);
    size_t need = 16 + CG_LOSS_MAX_G * 8 + (size_t)nchunks * G * 4;
    if (need > ws_bytes) {
        set_error("recon_head_fwd: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    launch_k(recon_head_fwd_kernel, nchunks * G, 256, 0, ST, h, x, sums, ws_part(ws), ws_counter(ws), G, npix, nchunks);
    return check_launch("recon_head_fwd");
}

extern "C" int cg_vgg_loss(const float* f_img, const float* mean_img, const float* rstd_img, const float* f_tgt, const float* mean_tgt,
                           const float* rstd_tgt, int R, int B, int per_dir, int HW, int C, float coef, float* sums, float* d_pre, void* ws,
                           size_t ws_bytes, void* stream) {
    CG_REQUIRE(f_img && mean_img && rstd_img && f_tgt && mean_tgt && rstd_tgt && sums && d_pre, "vgg_loss: NULL argument");
    CG_REQUIRE(R >= 1 && B >= 1 && per_dir >= B && per_dir % B == 0 && R % per_dir == 0 && HW >= 1 && C >= VL_CH && C % VL_CH == 0,
               "vgg_loss: R=%d B=%d per_dir=%d HW=%d C=%d out of range", R, B, per_dir, HW, C);
    const int nterm = R / B, nchunk = C / VL_CH;
    CG_REQUIRE(nterm <= 256, "vgg_loss: %d terms (R / B) exceed 256", nterm);
    const size_t need = 16 + CG_LOSS_MAX_G * 8 + (size_t)R * nchunk * 4;
    if (need > ws_bytes) {
        set_error("vgg_loss: workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    launch_k(vgg_loss_kernel, R * nchunk, 256, 0, ST, f_img, mean_img, rstd_img, f_tgt, mean_tgt, rstd_tgt, coef, d_pre, sums, ws_part(ws),
             ws_counter(ws), B, per_dir, HW, C, nterm);
    return check_launch("vgg_loss");
}

extern "C" int cg_recon_head_bwd(const float* h, const float* x, float coef, float* dh_pre, int G, int B, int HW, void* stream) {
    CG_REQUIRE(h && x && dh_pre && G >= 1 && B >= 1 && HW >= 1, "recon_head_bwd: G=%d B=%d HW=%d out of range", G, B, HW);
    const long npix = (long)B * HW, total = npix * G;
    launch_k(recon_head_bwd_kernel, cdiv(total, 256), 256, 0, ST, h, x, coef, dh_pre, total, npix);
    return check_launch("recon_head_bwd");
}
