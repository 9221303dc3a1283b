// TF32 implicit-GEMM convolution for sm_90a (TMA + mbarrier pipeline, warpgroup MMA).
//
//   D[128 pixels x BN couts] (fp32, registers) += A[128 x 32] (im2col tile of x, smem) * B[BN x 32] (weights, smem)
//
// * A tiles are gathered by TMA in IM2COL mode straight from the channels-last activation tensor
//   [G*B][H][W][Cin]: the zero padding of nn.ZeroPad2d (networks.py:473-474) is the TMA out-of-bound
//   fill, the stride is the TMA traversal stride -- there is no pad kernel and no im2col buffer.
// * B tiles are 2-D TMA boxes of the OHWI weight matrix [G*Cout][KH*KW*Cin] (K-major).
// * both land in shared memory in the 128-byte swizzled K-major layout wgmma reads; operands are
//   fp32 in HBM, converted to TF32 by the tensor map data type; accumulation is fp32 in registers.
// * warp-specialised persistent CTAs (one per SM): one producer thread issues the TMA loads, two consumer
//   warpgroups (64 pixel rows each) issue the MMAs and run the epilogue (bias / activation / addend / mask -> global).
//   smem ring of stages of (A,B) tiles with full/empty mbarriers.
// * all N council members are one launch: the member index is folded into the tensor-map coordinates
//   (image index g*B+n for A, row g*Cout+co for B), i.e. a grouped GEMM over the council.
//
// The same kernel serves the data gradient: the host passes dy as the activation, a transposed /
// flipped copy of the weights, and (for stride-2 layers) one launch "class" per output parity with its
// own im2col bounding box and a strided output mapping (see tc_conv_dgrad).
//
// Kernels in this file (host dispatch at the bottom of each section):
//   conv_tc_kernel<BK, BN>  forward / data gradient
//   wgrad_tc_kernel<BM, BN> weight gradient (MN-major operands transposed in shared memory, then wgmma)
//   wgrad_tma_kernel<BM, BN> weight gradient of stride-1 and stride-2 KxK layers (TMA-fed, shifted operand from registers)
//
// Reference call sites replaced: nn.Conv2d forward (networks.py:513,516) and cuDNN dgrad via autograd.
#include "common.cuh"
#include "tc_ptx.cuh"
#include <cstdlib>
#include <cstdio>
#include <cuda.h>
#include <mutex>
#include <string.h>

namespace cg {

// ------------------------------------------------------------------------------------------------
// driver entry points for tensor-map encoding (no link-time dependency on libcuda)
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*ReplaceAddressFn)(CUtensorMap*, void*);
static EncodeTiledFn g_encode_tiled = nullptr;
static ReplaceAddressFn g_replace_address = nullptr;
static EncodeIm2colFn g_encode_im2col = nullptr;
static int g_sm_count_dev[CG_MAX_DEVICES] = {0};  // multiprocessors per device ordinal
static int sm_count_now() {
    int dev = current_device();
    if (!g_sm_count_dev[dev]) cudaDeviceGetAttribute(&g_sm_count_dev[dev], cudaDevAttrMultiProcessorCount, dev);
    return g_sm_count_dev[dev];
}
thread_local int g_small_bn = 1;  // narrower N tiles when a launch has fewer tiles than SMs (mode bit 23 clears it)
thread_local int g_tc_serial_epilogue = 0;  // mode bit 26 sets it: conv_tc_kernel's previous epilogue and tile walk, for comparisons
thread_local int g_tc_reg_epilogue = 0;     // mode bit 27 sets it: every conv_tc_kernel launch on the register epilogue, for comparisons
static int g_driver_version = 0;
static std::once_flag g_once;

// ------------------------------------------------------------------------------------------------
// tensor-map cache (SURVEY 8b: "lazily-created TMA descriptor cache keyed by (ptr, shape), guarded by a mutex"): a training
// step issues ~1500 cuTensorMapEncode* calls, almost all of them for (address, geometry) pairs seen in the previous step (the
// caching allocator hands the same blocks out again); a direct-mapped table of encoded descriptors replaces the driver call by a
// 48-byte key comparison and a 128-byte copy.  The descriptor depends on nothing but the key, so a stale entry is impossible.
// ------------------------------------------------------------------------------------------------
struct MapKey {
    const void* ptr;
    int64_t a, b;      // leading sizes (rows / images, ktot, ...)
    int32_t v[8];      // remaining geometry: sizes, box, corners, stride, kind
    bool operator==(const MapKey& o) const { return ptr == o.ptr && a == o.a && b == o.b && memcmp(v, o.v, sizeof(v)) == 0; }
};
struct MapSlot {
    MapKey key;
    CUtensorMap map;
    bool used;
};
constexpr int MAP_SLOTS = 8192;
static MapSlot* g_map_cache = nullptr;
static std::mutex g_map_mutex;
static std::atomic<uint64_t> g_map_hits{0}, g_map_misses{0};
static inline uint32_t map_hash(const MapKey& k) {
    uint64_t h = 1469598103934665603ull;
    const unsigned char* p = reinterpret_cast<const unsigned char*>(&k);
    for (size_t i = 0; i < sizeof(MapKey); i++) h = (h ^ p[i]) * 1099511628211ull;
    return (uint32_t)(h ^ (h >> 32)) & (MAP_SLOTS - 1);
}
// encode(map) is called on a miss; returns its status
template <class F>
static int cached_map(CUtensorMap* out, const MapKey& key, F encode) {
    const uint32_t slot = map_hash(key);
    {
        std::lock_guard<std::mutex> lock(g_map_mutex);
        if (!g_map_cache) g_map_cache = new MapSlot[MAP_SLOTS]();
        MapSlot& s = g_map_cache[slot];
        if (s.used && s.key == key) {
            *out = s.map;
            g_map_hits.fetch_add(1, std::memory_order_relaxed);
            return CG_OK;
        }
    }
    if (int rc = encode(out)) return rc;
    g_map_misses.fetch_add(1, std::memory_order_relaxed);
    std::lock_guard<std::mutex> lock(g_map_mutex);
    MapSlot& s = g_map_cache[slot];
    s.key = key;
    s.map = *out;
    s.used = true;
    return CG_OK;
}
void tc_map_cache_stats(uint64_t* hits, uint64_t* misses) {
    *hits = g_map_hits.load();
    *misses = g_map_misses.load();
}

static void init_driver() {
    std::call_once(g_once, [] {
        cudaDriverEntryPointQueryResult q;
        void* fn = nullptr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            g_encode_tiled = (EncodeTiledFn)fn;
        fn = nullptr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            g_encode_im2col = (EncodeIm2colFn)fn;
        fn = nullptr;
        if (cudaGetDriverEntryPoint("cuTensorMapReplaceAddress", &fn, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            g_replace_address = (ReplaceAddressFn)fn;
        cudaDriverGetVersion(&g_driver_version);
    });
}

// ------------------------------------------------------------------------------------------------
// kernel
// ------------------------------------------------------------------------------------------------
constexpr int TC_BM = 128;          // pixels per tile
constexpr int TC_BK = 32;           // fp32 channels per stage = one 128-byte swizzle row
constexpr int TC_THREADS = 384;     // warpgroup 0: TMA producer (one thread); warpgroups 1, 2: wgmma + epilogue of tile rows 0..63 / 64..127
constexpr int TC_MAX_STAGES = 12;
constexpr int TC_MAX_CLASSES = 4;   // stride-2 dgrad: one im2col map per output parity class

struct TcClass {
    CUtensorMap amap;     // im2col map of the activation for this class
    int w0, h0;           // base coordinate of output pixel (0,0): lower corner
    int out_h0, out_w0;   // output pixel (p,q) is written to (p*out_sh + out_h0, q*out_sw + out_w0)
    int wrow_off;         // row offset into the weight matrix for this class
    int pad_;
};
struct TcParams {
    CUtensorMap bmap;               // weights [rows][Ktot_class] 2-D
    TcClass cls[TC_MAX_CLASSES];
    int ncls;
    int G, xg_images;               // groups; images per group in the activation map (0: shared input)
    int B, P, Q;                    // output grid per class: P x Q pixels per image
    int Cin, Cout, KH, KW, stride;  // KH,KW: taps per class
    int bn;                         // N tile
    int bk;                         // K elements per stage: 32 (128-byte swizzled rows) or 8 (32-byte rows, Cin = 8)
    int cps;                        // K chunks per pipeline stage
    int n_store;                    // output channels actually stored per N tile (== bn except the narrow image / head outputs)
    int out_H, out_W, out_sh, out_sw;  // full output spatial size and class strides
    int w_rows_per_group;           // weight rows per group (ncls * Cout for dgrad classes)
    float* y; const float* bias; const float* addend; const float* mask_src;
    float* stats;                   // optional [chunks][G*B*Cout][2] partial (sum, sum of squares) of the raw output, or NULL
    long stats_gbc;                 // G*B*Cout
    int act; float slope;
    int stages;
    int serial_epilogue;            // mode bit 26: addend and mask loaded one column group and row at a time, classes walked outermost
    // shared-memory epilogue (epi_slots > 0, chosen in launch_tc): 5-D tiled fp32 maps of y, the addend and the mask
    // (encode_out_map), a ring of epi_slots slots of epi_slot_bytes holding one 32-channel column slice of a tile
    CUtensorMap ymap, addmap, maskmap;
    int epi_slots, epi_slot_bytes;
};

// Tile t -> (pixel tile mt, N tile nt, class c, group g).  The classes of one pixel tile are neighbours in the walk, so the CTAs
// running them at the same time read overlapping im2col boxes of the same activation tile and all but the first find it in L2
// (class-outer, a stride-2 data gradient or upsample forward streams the whole activation from HBM once per class).
__device__ __forceinline__ void tc_tile(const TcParams& p, int t, int MT, int NT, int& mt, int& nt, int& c, int& g) {
    if (p.serial_epilogue) {
        mt = t % MT;
        int r = t / MT;
        nt = r % NT;
        r /= NT;
        c = r % p.ncls;
        g = r / p.ncls;
        return;
    }
    c = t % p.ncls;
    int r = t / p.ncls;
    mt = r % MT;
    r /= MT;
    nt = r % NT;
    g = r / NT;
}

// Coordinates in the 5-D view of the output (encode_out_map) of the 64 pixels h * 64 .. h * 64 + 63 of pixel tile mt: q = column
// of the first pixel in the class grid, n = image row index (g * B + img) * out_H / out_sh + row.  The shared-memory epilogue
// serves P * Q % 128 == 0 and (Q % 64 == 0 or 64 % Q == 0) only, so the 64 pixels are one row segment or whole rows of one image.
__device__ __forceinline__ void tc_half_coords(const TcParams& p, int g, int mt, int h, int& q, int& n) {
    const int pq = p.P * p.Q;
    const int m = mt * TC_BM + 64 * h;
    const int img = m / pq, rem = m - img * pq;
    const int pp = rem / p.Q;
    q = rem - pp * p.Q;
    n = (g * p.B + img) * (p.out_H / p.out_sh) + pp;
}

// Persistent CTAs (one per SM) walk the tiles (group, N tile, pixel tile, class; see tc_tile).  The producer thread streams (A, B) chunks
// through a ring of `stages` shared-memory slots guarded by full / empty mbarriers; each consumer warpgroup multiplies its 64
// pixel rows of A with the whole B tile (wgmma, accumulators in registers), releases a slot as soon as the MMAs that read it
// have retired, and runs the epilogue straight from registers while the producer already fills the slots of the next tile.
template <int BK, int BN>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const __grid_constant__ TcParams p) {
    pdl_trigger();
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0), tid = threadIdx.x & 127;  // warp-uniform for the compiler
    constexpr int a_bytes = TC_BM * BK * 4;                      // one K chunk of A
    constexpr int b_bytes = ((BN * BK * 4) + 1023) & ~1023;     // one K chunk of B (slot size)
    const int stage_bytes = p.cps * (a_bytes + b_bytes);         // [A_0..A_cps-1][B_0..B_cps-1]
    constexpr int tx_chunk = a_bytes + BN * BK * 4;
    constexpr bool tma_epi = BK == 32 && BN >= 64;  // the host sets epi_slots only for these instantiations
    const int epi_slots = tma_epi ? p.epi_slots : 0;
    uint8_t* epi = smem + (size_t)p.stages * stage_bytes;  // epilogue ring, 1024-byte aligned (stage_bytes is a multiple of 1024)
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(epi + (size_t)epi_slots * p.epi_slot_bytes);
    uint64_t* empty_bar = full_bar + p.stages;
    uint64_t* efull_bar = empty_bar + p.stages;
    uint64_t* eempty_bar = efull_bar + epi_slots;

    const int MT = (p.B * p.P * p.Q + TC_BM - 1) / TC_BM;  // pixel tiles per (group, class)
    const int NT = (p.Cout + BN - 1) / BN;
    const int tiles = p.G * p.ncls * NT * MT;
    const int kchunks = (p.Cin + BK - 1) / BK;  // a partial last chunk reads zero-filled channels
    const int kiters = p.KH * p.KW * kchunks;

    if (threadIdx.x == 0) {
        prefetch_tmap(&p.bmap);
        for (int c = 0; c < p.ncls; c++) prefetch_tmap(&p.cls[c].amap);
        for (int s = 0; s < p.stages; s++) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2);  // one arrival per consumer warpgroup
        }
        if (epi_slots) {
            prefetch_tmap(&p.ymap);
            if (p.addend) prefetch_tmap(&p.addmap);
            if (p.mask_src) prefetch_tmap(&p.maskmap);
        }
        for (int s = 0; s < epi_slots; s++) {
            mbar_init(&efull_bar[s], 1);
            mbar_init(&eempty_bar[s], 2);  // one arrival per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();  // on-chip prologue done: from here on the kernel reads what its predecessors in the stream wrote

    if (wg == 0) {
        // ===================== TMA producer =====================
        if (tid == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
                int mt, nt, c, g;
                tc_tile(p, t, MT, NT, mt, nt, c, g);
                const TcClass& cl = p.cls[c];
                long m0 = (long)mt * TC_BM;
                int img = (int)(m0 / (p.P * p.Q));
                int rem = (int)(m0 - (long)img * p.P * p.Q);
                int pp = rem / p.Q, qq = rem - pp * p.Q;
                int n_coord = g * p.xg_images + img;
                int w_coord = cl.w0 + qq * p.stride;
                int h_coord = cl.h0 + pp * p.stride;
                int wrow = g * p.w_rows_per_group + cl.wrow_off + nt * BN;
                int kh = 0, kw = 0, kc = 0;
                for (int k0 = 0; k0 < kiters; k0 += p.cps) {
                    const int n = kiters - k0 < p.cps ? kiters - k0 : p.cps;
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t* sa = smem + (size_t)stage * stage_bytes;
                    uint8_t* sb = sa + p.cps * a_bytes;
                    mbar_expect_tx(&full_bar[stage], (uint32_t)(n * tx_chunk));
                    for (int j = 0; j < n; j++) {
                        tma_load_im2col_4d(&cl.amap, &full_bar[stage], sa + j * a_bytes, kc * BK, w_coord, h_coord, n_coord, (uint16_t)kw,
                                           (uint16_t)kh);
                        tma_load_2d(&p.bmap, &full_bar[stage], sb + j * b_bytes, (kh * p.KW + kw) * p.Cin + kc * BK, wrow);
                        if (++kc == kchunks) { kc = 0; if (++kw == p.KW) { kw = 0; ++kh; } }
                    }
                    if (++stage == p.stages) { stage = 0; phase ^= 1; }
                }
            }
        } else if (tid == 32 && epi_slots) {
            // epilogue operands: the addend and mask slices of each tile's output region, one 32-channel slice per ring slot, each
            // as two 64-pixel boxes (one per consumer warpgroup).  Runs ahead of the consumers by the ring depth, i.e. during the
            // main loop of the tile; without operands the slot is only handed over as staging for the output.
            const uint32_t ebytes = (p.addend ? 2 * 8192 : 0) + (p.mask_src ? 2 * 8192 : 0);
            int es = 0;
            uint32_t ephase = 0;
            for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
                int mt, nt, c, g;
                tc_tile(p, t, MT, NT, mt, nt, c, g);
                const TcClass& cl = p.cls[c];
                int q[2], n[2];
                tc_half_coords(p, g, mt, 0, q[0], n[0]);
                tc_half_coords(p, g, mt, 1, q[1], n[1]);
                for (int sl = 0; sl < BN / 32; sl++) {
                    mbar_wait(&eempty_bar[es], ephase ^ 1);
                    if (ebytes) {
                        mbar_expect_tx(&efull_bar[es], ebytes);
                        uint8_t* dst = epi + (size_t)es * p.epi_slot_bytes;
                        const int c0 = nt * BN + 32 * sl;
                        for (int h = 0; h < 2; h++) {
                            if (p.addend) tma_load_5d(&p.addmap, &efull_bar[es], dst + h * 8192, c0, cl.out_w0, q[h], cl.out_h0, n[h]);
                            if (p.mask_src)
                                tma_load_5d(&p.maskmap, &efull_bar[es], dst + (p.addend ? 16384 : 0) + h * 8192, c0, cl.out_w0, q[h],
                                            cl.out_h0, n[h]);
                        }
                    } else {
                        mbar_arrive(&efull_bar[es]);
                    }
                    if (++es == epi_slots) { es = 0; ephase ^= 1; }
                }
            }
        }
        return;
    }

    // ===================== MMA + epilogue (consumer warpgroups) =====================
    const int cw = wg - 1;                                   // tile rows 64 cw .. 64 cw + 63
    const int warp4 = tid >> 5, lane = tid & 31;
    const int row0 = cw * 64 + warp4 * 16 + (lane >> 2);     // this thread's accumulator rows: row0, row0 + 8
    const int cq = 2 * (lane & 3);                           // ... and columns 8 j + cq, 8 j + cq + 1
    const uint64_t desc0 = BK == 32 ? make_kmajor_sw128_desc(0) : make_kmajor_sw32_desc(0);
    float acc[BN / 2];
    int stage = 0;
    uint32_t phase = 0;
    int es = 0;
    uint32_t ephase = 0;
    for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
        int mt, nt, c, g;
        tc_tile(p, t, MT, NT, mt, nt, c, g);
        const TcClass& cl = p.cls[c];
        int prev = -1;
        for (int k0 = 0; k0 < kiters; k0 += p.cps) {
            const int n = kiters - k0 < p.cps ? kiters - k0 : p.cps;
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sa = smem_u32(smem + (size_t)stage * stage_bytes) + cw * (64 * BK * 4);
            const uint32_t sb = smem_u32(smem + (size_t)stage * stage_bytes) + p.cps * a_bytes;
            wgmma_fence();
            for (int j = 0; j < n; j++) {
                const uint64_t adesc = desc0 | (uint64_t)(((sa + j * a_bytes) & 0x3FFFF) >> 4);
                const uint64_t bdesc = desc0 | (uint64_t)(((sb + j * b_bytes) & 0x3FFFF) >> 4);
#pragma unroll
                for (int kk = 0; kk < BK / 8; kk++)  // advance 8 tf32 (32 bytes) along K inside the swizzled row: +2 in the address field
                    wgmma_tf32<BN>(acc, adesc + (uint64_t)(kk * 2), bdesc + (uint64_t)(kk * 2), (k0 | j | kk) != 0 ? 1 : 0);
            }
            wgmma_commit();
            wgmma_wait<1>();  // the MMAs of the previous stage have retired: its slot can be refilled
            if (prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);
            prev = stage;
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_reg_fence(acc, BN / 2);
        if (tid == 0) mbar_arrive(&empty_bar[prev]);

        const int pq = p.P * p.Q;
        long out_off[2];
        bool valid[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int m = mt * TC_BM + row0 + 8 * h;  // < 2^31: B*P*Q pixels per member
            valid[h] = m < p.B * pq;
            out_off[h] = 0;
            if (valid[h]) {
                int img = m / pq;
                int rem = m - img * pq;
                int pp = rem / p.Q, qq = rem - pp * p.Q;
                long pix = ((long)(g * p.B + img) * p.out_H + (pp * p.out_sh + cl.out_h0)) * p.out_W + (qq * p.out_sw + cl.out_w0);
                out_off[h] = pix * p.Cout + nt * p.n_store;
            }
        }
        if (p.stats) {
            // instance-norm statistics of the raw convolution output, fused here instead of a second pass over y.  Every tile lies
            // inside one image (P*Q % 128 == 0); each warp reduces its 16 rows per column and writes one partial chunk.
            // The 8 lanes of a column pair (lane % 4) hold (s0, s1, q0, q1) each and are summed in pairs at lane distance 4, 8,
            // 16.  Transpose-reduce: at each level a lane keeps the half of its values that its lane bit selects and receives
            // the partner's part of that half, so the 4 values take 4 shuffles instead of 12.  Every sum adds the same two
            // operands as a plain butterfly (bits unchanged); lane l < 16 ends with element 2 * bit3 + bit2 of (s0, q0, s1, q1).
            const int tiles_per_img = pq / TC_BM;
            const int img = (mt * TC_BM) / pq;
            const int chunk = ((c * tiles_per_img + (mt - img * tiles_per_img)) << 3) + cw * 4 + warp4;
            const bool b2 = lane & 4, b3 = lane & 8;
            float* st = p.stats + ((long)chunk * p.stats_gbc + (long)(g * p.B + img) * p.Cout + nt * BN + cq) * 2 + (b3 ? 2 : 0) + (b2 ? 1 : 0);
#pragma unroll
            for (int j = 0; j < BN / 8; j++) {
                const float s0 = acc[4 * j] + acc[4 * j + 2], s1 = acc[4 * j + 1] + acc[4 * j + 3];
                const float q0 = acc[4 * j] * acc[4 * j] + acc[4 * j + 2] * acc[4 * j + 2];
                const float q1 = acc[4 * j + 1] * acc[4 * j + 1] + acc[4 * j + 3] * acc[4 * j + 3];
                // level 4: keep (s0, s1) or (q0, q1)
                const float k0 = b2 ? q0 : s0, k1 = b2 ? q1 : s1;
                const float r0 = __shfl_xor_sync(0xffffffffu, b2 ? s0 : q0, 4), r1 = __shfl_xor_sync(0xffffffffu, b2 ? s1 : q1, 4);
                const float x0 = k0 + r0, x1 = k1 + r1;
                // level 8: keep column cq or cq + 1
                float v = (b3 ? x1 : x0) + __shfl_xor_sync(0xffffffffu, b3 ? x0 : x1, 8);
                // level 16
                v += __shfl_xor_sync(0xffffffffu, v, 16);
                if (lane < 16) st[16 * j] = v;
            }
        }
        if constexpr (tma_epi) {
            if (epi_slots) {
                // Shared-memory epilogue, one 32-channel column slice at a time: combine the accumulators with the slice's operands,
                // which the operand thread loaded during the main loop, write the result over the first operand (or into the empty
                // slot), and store this warpgroup's 64 x 32 half with one TMA store.  Same operations per element, in the same
                // order, as the register epilogue below.  The slot goes back to the operand thread once the store has read it.
                int q, n;
                tc_half_coords(p, g, mt, cw, q, n);
                const int r0 = warp4 * 16 + (lane >> 2);  // this thread's rows of the warpgroup's 64-pixel half: r0, r0 + 8
#pragma unroll
                for (int sl = 0; sl < BN / 32; sl++) {
                    float2 bv[4];
#pragma unroll
                    for (int jj = 0; jj < 4; jj++)
                        bv[jj] = p.bias ? __ldg(reinterpret_cast<const float2*>(p.bias + (long)g * p.Cout + nt * BN + 32 * sl + 8 * jj + cq))
                                        : make_float2(0.f, 0.f);
                    mbar_wait(&efull_bar[es], ephase);
                    uint8_t* half = epi + (size_t)es * p.epi_slot_bytes + cw * 8192;  // [64 pixels][32 channels], 128-byte swizzle
                    const uint8_t* msk = half + (p.addend ? 16384 : 0);
#pragma unroll
                    for (int jj = 0; jj < 4; jj++) {
                        const int j = 4 * sl + jj;
#pragma unroll
                        for (int h = 0; h < 2; h++) {
                            const int r = r0 + 8 * h;
                            const int off = r * 128 + (((2 * jj + (cq >> 2)) ^ (r & 7)) << 4) + (cq & 3) * 4;
                            float2 o = make_float2(acc[4 * j + 2 * h] + bv[jj].x, acc[4 * j + 2 * h + 1] + bv[jj].y);
                            if (p.addend) {
                                const float2 a = *reinterpret_cast<const float2*>(half + off);
                                o.x += a.x; o.y += a.y;
                            }
                            if (p.mask_src) {
                                const float2 a = *reinterpret_cast<const float2*>(msk + off);
                                o.x *= a.x > 0.f ? 1.f : p.slope; o.y *= a.y > 0.f ? 1.f : p.slope;
                            } else if (p.act != CG_ACT_NONE) {
                                o.x = apply_act(o.x, p.act, p.slope); o.y = apply_act(o.y, p.act, p.slope);
                            }
                            *reinterpret_cast<float2*>(half + off) = o;
                        }
                    }
                    fence_proxy_async();  // the generic-proxy writes above are visible to the TMA store
                    named_bar_sync(1 + cw, 128);
                    if (tid == 0) {
                        tma_store_5d(&p.ymap, half, nt * BN + 32 * sl, cl.out_w0, q, cl.out_h0, n);
                        bulk_commit();
                        // hand back the previous slice's slot once its store has read it (this one's is still in flight); the
                        // last slice of the tile waits for its own, so that the next tile's operands can be loaded during its main loop
                        if (sl > 0) {
                            bulk_wait_read<1>();
                            mbar_arrive(&eempty_bar[es == 0 ? epi_slots - 1 : es - 1]);
                        }
                        if (sl == BN / 32 - 1) {
                            bulk_wait_read<0>();
                            mbar_arrive(&eempty_bar[es]);
                        }
                    }
                    if (++es == epi_slots) { es = 0; ephase ^= 1; }
                }
                continue;
            }
        }
        // each row's 8-column group is written by four consecutive lanes: 32 contiguous bytes, one full sector
        if (!(p.addend || p.mask_src) || p.serial_epilogue) {
#pragma unroll
            for (int j = 0; j < BN / 8; j++) {
                const int col = 8 * j + cq;
                if (col >= p.n_store) break;
                float2 bv = make_float2(0.f, 0.f);
                if (p.bias) bv = __ldg(reinterpret_cast<const float2*>(p.bias + (long)g * p.Cout + nt * p.n_store + col));
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    if (!valid[h]) continue;
                    float2 o = make_float2(acc[4 * j + 2 * h] + bv.x, acc[4 * j + 2 * h + 1] + bv.y);
                    if (p.addend) {
                        const float2 a = __ldg(reinterpret_cast<const float2*>(p.addend + out_off[h] + col));
                        o.x += a.x; o.y += a.y;
                    }
                    if (p.mask_src) {
                        const float2 a = __ldg(reinterpret_cast<const float2*>(p.mask_src + out_off[h] + col));
                        o.x *= a.x > 0.f ? 1.f : p.slope; o.y *= a.y > 0.f ? 1.f : p.slope;
                    } else if (p.act != CG_ACT_NONE) {
                        o.x = apply_act(o.x, p.act, p.slope); o.y = apply_act(o.y, p.act, p.slope);
                    }
                    *reinterpret_cast<float2*>(p.y + out_off[h] + col) = o;
                }
            }
            continue;
        }
        // Data gradient with a residual addend and / or an activation mask (no bias, no activation: tc_conv_dgrad never sets
        // them).  The compiler cannot prove that y aliases neither operand, so in the loop above it keeps every load behind the
        // previous store: a tile waits for BN / 4 global round trips in a row while the tensor cores idle.  Here the operands of
        // EB column groups are all loaded before the first of their results is stored: one round trip per batch.  EB is bounded
        // by the registers left beside the BN / 2 accumulators.
        constexpr int EB = BN == 256 ? 2 : BN / 8 < 8 ? BN / 8 : 8;
#pragma unroll
        for (int j0 = 0; j0 < BN / 8; j0 += EB) {
            float2 av[EB][2], mv[EB][2];
#pragma unroll
            for (int jj = 0; jj < EB; jj++) {
                const int col = 8 * (j0 + jj) + cq;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const bool ld = col < p.n_store && valid[h];
                    av[jj][h] = p.addend && ld ? __ldg(reinterpret_cast<const float2*>(p.addend + out_off[h] + col)) : make_float2(0.f, 0.f);
                    mv[jj][h] = p.mask_src && ld ? __ldg(reinterpret_cast<const float2*>(p.mask_src + out_off[h] + col)) : make_float2(0.f, 0.f);
                }
            }
#pragma unroll
            for (int jj = 0; jj < EB; jj++) {
                const int j = j0 + jj, col = 8 * j + cq;
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    if (col >= p.n_store || !valid[h]) continue;
                    // + 0: the zero bias of the loop above, which turns an accumulator of -0 into +0
                    float2 o = make_float2(acc[4 * j + 2 * h] + 0.f, acc[4 * j + 2 * h + 1] + 0.f);
                    if (p.addend) { o.x += av[jj][h].x; o.y += av[jj][h].y; }
                    if (p.mask_src) { o.x *= mv[jj][h].x > 0.f ? 1.f : p.slope; o.y *= mv[jj][h].y > 0.f ? 1.f : p.slope; }
                    *reinterpret_cast<float2*>(p.y + out_off[h] + col) = o;
                }
            }
        }
    }
    if (epi_slots && tid == 0) bulk_wait<0>();  // the TMA stores of y have completed before the CTA exits
}


// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static int encode_weights_map_raw(CUtensorMap* map, const float* w, long rows, long ktot, int bn, int bk) {
    cuuint64_t dims[2] = {(cuuint64_t)ktot, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ktot * 4};
    cuuint32_t box[2] = {(cuuint32_t)bk, (cuuint32_t)bn};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode_tiled(map, CU_TENSOR_MAP_DATA_TYPE_TFLOAT32, 2, (void*)w, dims, strides, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, bk == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_32B,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled(weights rows=%ld ktot=%ld bn=%d) failed: %d", rows, ktot, bn, (int)r);
        return CG_ERR_CUDA;
    }
    return CG_OK;
}

static int encode_weights_map(CUtensorMap* map, const float* w, long rows, long ktot, int bn, int bk = TC_BK) {
    MapKey k{};
    k.ptr = w; k.a = rows; k.b = ktot; k.v[0] = bn; k.v[1] = bk; k.v[7] = 1;
    return cached_map(map, k, [&](CUtensorMap* m) { return encode_weights_map_raw(m, w, rows, ktot, bn, bk); });
}

static int encode_weights_map_p(TcParams& p, const float* w, long rows, long ktot) {
    return encode_weights_map(&p.bmap, w, rows, ktot, p.bn, p.bk);
}

// activation [N][H][W][C] viewed by TMA as (C, W, H, N); bounding box corners as in CUTLASS
// (cutlass/conv/collective/detail.hpp compute_lower/upper_corner_whd): lower = -pad_lo, upper = pad_hi - (K-1).
static int encode_act_map_raw(CUtensorMap* map, const float* x, long N, int H, int W, int C, int lo_w, int lo_h, int up_w, int up_h,
                              int stride, int bk) {
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    cuuint64_t strides[3] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4};
    int lower[2] = {lo_w, lo_h};
    int upper[2] = {up_w, up_h};
    cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    CUresult r = g_encode_im2col(map, CU_TENSOR_MAP_DATA_TYPE_TFLOAT32, 4, (void*)x, dims, strides, lower, upper, bk, TC_BM, estr,
                                 CU_TENSOR_MAP_INTERLEAVE_NONE, bk == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_32B,
                                 CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeIm2col(N=%ld H=%d W=%d C=%d corners %d,%d / %d,%d stride %d) failed: %d", N, H, W, C, lo_w, lo_h,
                  up_w, up_h, stride, (int)r);
        return CG_ERR_CUDA;
    }
    // driver <= 13.1: small tensors need bit 21 of the second descriptor word cleared (same workaround as CUTLASS
    // cute/atom/copy_traits_sm90_im2col.hpp:477-483)
    if (g_driver_version <= 13010 && (long)N * H * W * C * 4 < 131072) reinterpret_cast<uint64_t*>(map)[1] &= ~(1ull << 21);
    return CG_OK;
}

static int encode_act_map(CUtensorMap* map, const float* x, long N, int H, int W, int C, int lo_w, int lo_h, int up_w, int up_h,
                          int stride, int bk = TC_BK) {
    MapKey k{};
    k.ptr = x; k.a = N; k.b = ((int64_t)H << 32) | (uint32_t)W;
    k.v[0] = C; k.v[1] = lo_w; k.v[2] = lo_h; k.v[3] = up_w; k.v[4] = up_h; k.v[5] = stride; k.v[6] = bk; k.v[7] = 2;
    return cached_map(map, k, [&](CUtensorMap* m) { return encode_act_map_raw(m, x, N, H, W, C, lo_w, lo_h, up_w, up_h, stride, bk); });
}

// Output-shaped tensor [NI][H][W][C] (y, the addend, the mask) for the shared-memory epilogue, viewed as 5-D (C, sw, W / sw, sh,
// NI * H / sh): pixel (p, q) of the output class (h0, w0) with strides (sh, sw) is (c, w0, q, h0, n * H / sh + p), so the class
// strides are plain coordinates and no TMA traversal stride is involved.  Box: 32 channels (one 128-byte swizzled row) x 64
// pixels, qbox of one row x 64 / qbox rows.  FLOAT32: the values move raw, unlike the TF32 operand maps.  The descriptor is cached
// by geometry alone and pointed at `t` by cuTensorMapReplaceAddress: outputs are often fresh allocations (a layer's y is), and
// replacing the address costs far less than an encode.
static int encode_out_map(CUtensorMap* map, const float* t, long NI, int H, int W, int C, int sh, int sw, int qbox) {
    MapKey k{};
    k.ptr = nullptr; k.a = NI; k.b = ((int64_t)H << 32) | (uint32_t)W;
    k.v[0] = C; k.v[1] = sh; k.v[2] = sw; k.v[3] = qbox; k.v[7] = 3;
    if (int rc = cached_map(map, k, [&](CUtensorMap* m) {
            cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)sw, (cuuint64_t)(W / sw), (cuuint64_t)sh, (cuuint64_t)(NI * H / sh)};
            cuuint64_t strides[4] = {(cuuint64_t)C * 4, (cuuint64_t)sw * C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)sh * W * C * 4};
            cuuint32_t box[5] = {32, 1, (cuuint32_t)qbox, 1, (cuuint32_t)(64 / qbox)};
            cuuint32_t estr[5] = {1, 1, 1, 1, 1};
            CUresult r = g_encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, (void*)t, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) {
                set_error("cuTensorMapEncodeTiled(output NI=%ld H=%d W=%d C=%d strides %d,%d box q %d) failed: %d", NI, H, W, C, sh, sw, qbox, (int)r);
                return CG_ERR_CUDA;
            }
            return CG_OK;
        }))
        return rc;
    CUresult r = g_replace_address(map, (void*)t);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapReplaceAddress(output NI=%ld H=%d W=%d C=%d) failed: %d", NI, H, W, C, (int)r);
        return CG_ERR_CUDA;
    }
    return CG_OK;
}

static int pick_bn(int cout) {
    if (cout % 256 == 0) return 256;
    if (cout == 128) return 128;
    if (cout == 64) return 64;
    if (cout <= 16 && cout % 4 == 0) return 16;  // narrow outputs: 16 accumulator columns, `cout` stored
    return 0;
}
// K elements per pipeline stage: 32-channel (128-byte) rows, or 8-channel (32-byte) rows for <= 16 channels
static int pick_bk(int cin) {
    if (cin % TC_BK == 0) return TC_BK;
    if (cin <= 16 && cin % 4 == 0) return 8;
    return 0;
}

// Few-tile launches (small maps: the 32x32 bottleneck of the 128x128 configuration is 8 pixel tiles per member): narrower N tiles put more
// SMs to work.  Every extra N tile re-reads the same activation tile, from L2, which is cheap at these sizes; a 3x3 256->256 layer on
// 1024 pixels x 2 members goes from 16 CTAs running 288 K-steps of 256-wide MMAs to 64 CTAs running the same steps 64 wide.
static int fill_bn(int bn, long mpix, int groups_classes, int cout) {
    if (!g_small_bn) return bn;
    const int sms = sm_count_now();
    while (bn > 64 && cout % (bn / 2) == 0 && (long)groups_classes * cdiv(mpix, TC_BM) * (cout / bn) < sms) bn >>= 1;
    return bn;
}

bool tc_fwd_supported(const cg_conv_geom& g) {
    init_driver();
    if (!g_encode_tiled || !g_encode_im2col) return false;
    if (g.ups && !(g.KH == 3 && g.KW == 3 && g.stride == 1 && g.pad == 1 && g.Cin % TC_BK == 0)) return false;
    if (pick_bk(g.Cin) == 0) return false;
    if (pick_bn(g.Cout) == 0) return false;
    if (g.pad > 120 || g.KH > 120) return false;
    if ((long)g.B * (g.ups ? g.H * g.W : g.Ho * g.Wo) < TC_BM) return false;  // tiny maps: the SIMT kernel is fine
    return true;
}

template <int BK>
static void (*tc_kernel_for(int bn))(TcParams) {
    switch (bn) {
        case 16: return conv_tc_kernel<BK, 16>;
        case 64: return conv_tc_kernel<BK, 64>;
        case 128: return conv_tc_kernel<BK, 128>;
        case 256: return conv_tc_kernel<BK, 256>;
    }
    return nullptr;
}

static int launch_tc(TcParams& p, cudaStream_t st) {
    int a_bytes = TC_BM * p.bk * 4, b_bytes = ((p.bn * p.bk * 4) + 1023) & ~1023;
    int chunk_bytes = a_bytes + b_bytes;
    // several K chunks per stage when a chunk carries little tensor work (N <= 64 or 32-byte rows): fewer barrier round trips.  At
    // N = 128 one chunk per stage (6 or 7 stages of 32 KB instead of 3 of 64 KB) measured 8-18 % faster on the production launches.
    int kiters = p.KH * p.KW * ((p.Cin + p.bk - 1) / p.bk);
    int cps = p.bn <= 64 ? 2 : 1;
    if (p.bk == 8) cps = 8;          // 6 KB chunks
    while (cps > 1 && (cps > kiters || cps * chunk_bytes > 64 * 1024)) cps >>= 1;
    p.cps = cps;
    int stage_bytes = cps * chunk_bytes;
    int stages = (226 * 1024 - 1024 - 2 * TC_MAX_STAGES * 8) / stage_bytes;  // 227 KB dynamic shared memory per block
    if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
    if (stages > 4 && stage_bytes >= 48 * 1024) stages = 4;
    if (p.n_store == 0) p.n_store = p.bn;
    p.serial_epilogue = g_tc_serial_epilogue;
    // Shared-memory epilogue (TMA-loaded operands, TMA-stored results) where each 64-pixel half tile is a row segment or whole rows
    // of one image (tc_half_coords) and at least two ring slots fit beside the stages; elsewhere the register epilogue.  Slot: one
    // 16 KB [128 pixels][32 channels] slice per operand (the result overwrites the first), or a bare staging slice.
    p.epi_slots = 0;
    const int nops = (p.addend ? 1 : 0) + (p.mask_src ? 1 : 0);
    const bool aligned = ((uintptr_t)p.y | (uintptr_t)p.addend | (uintptr_t)p.mask_src) % 16 == 0;
    if (g_replace_address && !g_tc_reg_epilogue && !p.serial_epilogue && p.bk == TC_BK && p.bn >= 64 && p.n_store == p.bn && (long)p.P * p.Q % TC_BM == 0 &&
        (p.Q % 64 == 0 || 64 % p.Q == 0) && p.out_H % p.out_sh == 0 && p.out_W % p.out_sw == 0 && p.Cout % 4 == 0 && aligned) {
        const int slot_bytes = (nops ? nops : 1) * 16384;
        auto slots_beside = [&](int st) { return (int)((227L * 1024 - 1024 - (long)st * stage_bytes - 2 * st * 8) / (slot_bytes + 16)); };
        while (slots_beside(stages) < 2 && stages > 4) stages--;  // short-K launches: the stages past 4 buy nothing
        const int e = slots_beside(stages);
        if (e >= 2) {
            p.epi_slots = e < 4 ? e : 4;
            p.epi_slot_bytes = slot_bytes;
            const long ni = (long)p.G * p.B;
            const int qbox = p.Q < 64 ? p.Q : 64;
            if (int rc = encode_out_map(&p.ymap, p.y, ni, p.out_H, p.out_W, p.Cout, p.out_sh, p.out_sw, qbox)) return rc;
            if (p.addend)
                if (int rc = encode_out_map(&p.addmap, p.addend, ni, p.out_H, p.out_W, p.Cout, p.out_sh, p.out_sw, qbox)) return rc;
            if (p.mask_src)
                if (int rc = encode_out_map(&p.maskmap, p.mask_src, ni, p.out_H, p.out_W, p.Cout, p.out_sh, p.out_sw, qbox)) return rc;
        }
    }
    p.stages = stages;
    size_t smem = (size_t)stages * stage_bytes + 1024 /*align slack*/ + 2 * stages * 8 + (size_t)p.epi_slots * (p.epi_slot_bytes + 16);
    void (*kern)(TcParams) = p.bk == 32 ? tc_kernel_for<32>(p.bn) : tc_kernel_for<8>(p.bn);
    if (!kern) {
        set_error("conv_tc: no kernel for N tile %d / K chunk %d", p.bn, p.bk);
        return CG_ERR_ARG;
    }
    static PerDeviceOnce attr_set;
    if (attr_set.first()) {
        for (int bn : {16, 64, 128, 256}) {
            cudaError_t e = cudaFuncSetAttribute(tc_kernel_for<32>(bn), cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
            if (e == cudaSuccess) e = cudaFuncSetAttribute(tc_kernel_for<8>(bn), cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
            if (e != cudaSuccess) {
                attr_set.reset();
                set_error("cudaFuncSetAttribute(conv_tc_kernel): %s", cudaGetErrorString(e));
                return CG_ERR_CUDA;
            }
        }
    }
    int MT = cdiv((long)p.B * p.P * p.Q, TC_BM);
    long tiles = (long)p.G * p.ncls * ((p.Cout + p.bn - 1) / p.bn) * MT;
    const long slots = sm_count_now();
    int grid = (int)(tiles < slots ? tiles : slots);
    launch_k(kern, grid, TC_THREADS, smem, st, p);
    return check_launch("conv_tc_kernel");
}


// nearest-upsample x2 followed by a 3x3 pad-1 convolution == four 2x2 convolutions on the ORIGINAL tensor, one per
// output parity (a,b): output row 2i+a reads source rows {i-1,i} (a=0) or {i,i+1} (a=1), and the 3 filter rows
// collapse onto those 2 source rows: a=0 -> {w0, w1+w2}, a=1 -> {w0+w1, w2} (same along columns).  2.25x fewer
// FLOPs than convolving the materialised upsampled tensor, and the upsampled tensor never exists.
__global__ void ups_weight_transform_kernel(const float* __restrict__ w, float* __restrict__ wc, long total, int Cout, int Cin) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;  // wc[g][cls][co][r][s][ci]
    if (i >= total) return;
    int ci = (int)(i % Cin);
    long t = i / Cin;
    int ss = (int)(t % 2); t /= 2;
    int r = (int)(t % 2); t /= 2;
    int co = (int)(t % Cout); t /= Cout;
    int cls = (int)(t % 4);
    int g = (int)(t / 4);
    int a = cls >> 1, b = cls & 1;
    // taps of the 3-wide filter that land on source offset r for parity a
    int kh0 = a == 0 ? (r == 0 ? 0 : 1) : (r == 0 ? 0 : 2), kh1 = a == 0 ? (r == 0 ? 0 : 2) : (r == 0 ? 1 : 2);
    int kw0 = b == 0 ? (ss == 0 ? 0 : 1) : (ss == 0 ? 0 : 2), kw1 = b == 0 ? (ss == 0 ? 0 : 2) : (ss == 0 ? 1 : 2);
    const float* wp = w + ((long)g * Cout + co) * 9 * Cin + ci;
    float acc = 0.f;
    for (int kh = kh0; kh <= kh1; kh++)
        for (int kw = kw0; kw <= kw1; kw++) acc += __ldg(wp + (kh * 3 + kw) * Cin);
    wc[i] = acc;
}

size_t tc_fwd_ws(const cg_conv_geom& g) {
    return g.ups ? (size_t)g.G * 4 * g.Cout * 4 * g.Cin * sizeof(float) : 0;
}

// number of partial-statistics chunks the fused epilogue writes per (image, channel); 0: fusion not possible
int tc_fwd_stats_chunks(const cg_conv_geom& g) {
    if (pick_bn(g.Cout) < 32) return 0;
    long pq = g.ups ? (long)g.H * g.W : (long)g.Ho * g.Wo;
    if (pq % TC_BM != 0) return 0;
    return (int)((g.ups ? 4 : 1) * (pq / TC_BM) * 8);  // one chunk per consumer warp and tile
}

int tc_conv_fwd(const cg_conv_geom& g, const float* x, const float* w, const float* bias, float* y, int act, float slope, void* ws,
                size_t ws_bytes, cudaStream_t st, float* stats_part) {
    init_driver();
    TcParams p{};
    p.stats = stats_part;
    p.stats_gbc = (long)g.G * g.B * g.Cout;
    p.bn = pick_bn(g.Cout);
    if (p.bn > 64) p.bn = fill_bn(p.bn, (long)g.B * (g.ups ? g.H * g.W : g.Ho * g.Wo), g.G * (g.ups ? 4 : 1), g.Cout);
    p.n_store = p.bn == 16 ? g.Cout : p.bn;
    p.bk = pick_bk(g.Cin);
    long nimg = (long)(g.x_groups == 1 ? 1 : g.G) * g.B;
    p.G = g.G; p.xg_images = g.x_groups == 1 ? 0 : g.B;
    p.B = g.B; p.Cin = g.Cin; p.Cout = g.Cout;
    p.y = y; p.bias = bias; p.addend = nullptr; p.mask_src = nullptr; p.act = act; p.slope = slope;
    if (g.ups) {
        size_t need = tc_fwd_ws(g);
        if (need > ws_bytes) {
            set_error("conv_fwd(tc, upsample classes): workspace %zu < %zu bytes", ws_bytes, need);
            return CG_ERR_WORKSPACE;
        }
        float* wc = (float*)ws;
        long total = (long)g.G * 4 * g.Cout * 4 * g.Cin;
        launch_k(ups_weight_transform_kernel, cdiv(total, 256), 256, 0, st, w, wc, total, g.Cout, g.Cin);
        if (int rc = check_launch("ups_weight_transform")) return rc;
        if (int rc = encode_weights_map_p(p, wc, (long)g.G * 4 * g.Cout, 4L * g.Cin)) return rc;
        for (int c = 0; c < 4; c++) {
            int a = c >> 1, b = c & 1;
            int lo_h = a == 0 ? -1 : 0, lo_w = b == 0 ? -1 : 0;  // lower corner = -(left pad); upper = right pad - (K-1), K = 2
            int up_h = a == 0 ? -1 : 0, up_w = b == 0 ? -1 : 0;
            if (int rc = encode_act_map(&p.cls[c].amap, x, nimg, g.H, g.W, g.Cin, lo_w, lo_h, up_w, up_h, 1, p.bk)) return rc;
            p.cls[c].w0 = lo_w; p.cls[c].h0 = lo_h; p.cls[c].out_h0 = a; p.cls[c].out_w0 = b; p.cls[c].wrow_off = c * g.Cout;
        }
        p.ncls = 4;
        p.P = g.H; p.Q = g.W; p.KH = 2; p.KW = 2; p.stride = 1;
        p.out_H = g.Ho; p.out_W = g.Wo; p.out_sh = 2; p.out_sw = 2;
        p.w_rows_per_group = 4 * g.Cout;
        return launch_tc(p, st);
    }
    long ktot = (long)g.KH * g.KW * g.Cin;
    if (int rc = encode_weights_map_p(p, w, (long)g.G * g.Cout, ktot)) return rc;
    if (int rc = encode_act_map(&p.cls[0].amap, x, nimg, g.H, g.W, g.Cin, -g.pad, -g.pad, g.pad - (g.KW - 1), g.pad - (g.KH - 1), g.stride,
                                p.bk))
        return rc;
    p.cls[0].w0 = -g.pad; p.cls[0].h0 = -g.pad; p.cls[0].out_h0 = 0; p.cls[0].out_w0 = 0; p.cls[0].wrow_off = 0;
    p.ncls = 1;
    p.P = g.Ho; p.Q = g.Wo;
    p.KH = g.KH; p.KW = g.KW; p.stride = g.stride;
    p.out_H = g.Ho; p.out_W = g.Wo; p.out_sh = 1; p.out_sw = 1;
    p.w_rows_per_group = g.Cout;
    return launch_tc(p, st);
}

// ------------------------------------------------------------------------------------------------
// data gradient on the same kernel
//
// dx[ih] = sum_kh dy[(ih + pad - kh)/s] * w[kh]  over the kh with (ih + pad - kh) % s == 0.
// For the input-parity class ph = (ih + pad) % s only kh = ph + s*t, t < T = K/s, contribute, and with
// ih = ihf + s*i the sum is a T-tap stride-1 convolution over dy:
//     dx[ihf + s*i] = sum_r dy[i - padl + r] * w[ph + s*(T-1-r)],   padl = (T-1) - (ihf + pad - ph)/s
// so each class is a forward convolution of dy with transposed+flipped weights wt[g][class][ci][r][s][co],
// an im2col box with lower corner -padl, and an output written with stride s at offset ihf.
// ------------------------------------------------------------------------------------------------
// CinP >= Cin: rows ci >= Cin are zero (pads the 8 image lanes to the 16-wide N tile of the narrow kernels)
// 32 (co) x 32 (ci) tiles through shared memory: reads run along ci (contiguous in OHWI), writes along co (contiguous in the
// transposed copy); grid = (co tiles x ci tiles, KH*KW, G)
__global__ void __launch_bounds__(256) dgrad_weight_transform_kernel(const float* __restrict__ w, float* __restrict__ wt, int Cout, int Cin,
                                                                     int CinP, int KH, int KW, int s) {
    pdl_trigger();
    pdl_wait();
    __shared__ float tile[32][33];
    const int TH = KH / s, TW = KW / s;
    const int cit = (CinP + 31) / 32;
    const int co0 = (blockIdx.x / cit) * 32, ci0 = (blockIdx.x % cit) * 32;
    int t = blockIdx.y;
    const int ss = t % TW; t /= TW;
    const int r = t % TH; t /= TH;
    const int cls = t;
    const int g = blockIdx.z;
    const int ph = cls / s, pw = cls - ph * s;
    const int kh = ph + s * (TH - 1 - r), kw = pw + s * (TW - 1 - ss);
    const int tx = threadIdx.x, ty = threadIdx.y;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int co = co0 + ty + 8 * j, ci = ci0 + tx;
        tile[ty + 8 * j][tx] = (co < Cout && ci < Cin) ? __ldg(w + ((((long)g * Cout + co) * KH + kh) * KW + kw) * Cin + ci) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int ci = ci0 + ty + 8 * j, co = co0 + tx;
        if (ci < CinP && co < Cout) wt[(((((long)g * s * s + cls) * CinP + ci) * TH + r) * TW + ss) * Cout + co] = tile[tx][ty + 8 * j];
    }
}

bool tc_dgrad_supported(const cg_conv_geom& g) {
    init_driver();
    if (!g_encode_tiled || !g_encode_im2col) return false;
    int s = g.stride;
    if (s > 2 || g.KH % s || g.KW % s) return false;
    if (pick_bk(g.Cout) == 0) return false;   // K dimension of the dgrad GEMM
    if (pick_bn(g.Cin) == 0) return false;    // N dimension (<= 16 image / head lanes are padded to 16)
    int Hin = g.ups ? 2 * g.H : g.H, Win = g.ups ? 2 * g.W : g.W;
    if (Hin % s || Win % s) return false;
    if ((long)g.B * (Hin / s) * (Win / s) < TC_BM) return false;
    return true;
}

size_t tc_dgrad_ws(const cg_conv_geom& g) {
    size_t wt = (size_t)g.G * g.Cout * g.KH * g.KW * (g.Cin <= 16 ? 16 : g.Cin) * sizeof(float);
    wt = (wt + 1023) & ~(size_t)1023;
    size_t up = g.ups ? (size_t)g.G * g.B * 4 * g.H * g.W * g.Cin * sizeof(float) : 0;
    return wt + up;
}

int tc_conv_dgrad(const cg_conv_geom& g, const float* dy, const float* w, float* dx, const float* addend, const float* mask_src,
                  float mask_slope, void* ws, size_t ws_bytes, cudaStream_t st) {
    init_driver();
    size_t need = tc_dgrad_ws(g);
    if (need > ws_bytes) {
        set_error("conv_dgrad(tc): workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    const int s = g.stride, TH = g.KH / s, TW = g.KW / s, ncls = s * s;
    const int Hin = g.ups ? 2 * g.H : g.H, Win = g.ups ? 2 * g.W : g.W;
    float* wt = (float*)ws;
    const int CinP = g.Cin <= 16 ? 16 : g.Cin;
    size_t wt_bytes = ((size_t)g.G * g.Cout * g.KH * g.KW * CinP * sizeof(float) + 1023) & ~(size_t)1023;
    float* d_seen = g.ups ? (float*)((uint8_t*)ws + wt_bytes) : dx;
    long total = (long)g.G * g.Cout * g.KH * g.KW * CinP;
    (void)total;
    launch_k(dgrad_weight_transform_kernel, dim3(cdiv(g.Cout, 32) * cdiv(CinP, 32), g.KH * g.KW, g.G), dim3(32, 8), 0, st, w, wt, g.Cout, g.Cin, CinP,
                                                                                                                  g.KH, g.KW, s);
    if (int rc = check_launch("dgrad_weight_transform")) return rc;

    TcParams p{};
    p.bn = pick_bn(g.Cin);
    if (p.bn > 64) p.bn = fill_bn(p.bn, (long)g.B * ((g.ups ? 2 * g.H : g.H) / g.stride) * ((g.ups ? 2 * g.W : g.W) / g.stride), g.G * g.stride * g.stride, g.Cin);
    p.n_store = p.bn == 16 ? g.Cin : p.bn;
    p.bk = pick_bk(g.Cout);
    long ktot = (long)TH * TW * g.Cout;
    if (int rc = encode_weights_map_p(p, wt, (long)g.G * ncls * CinP, ktot)) return rc;
    for (int c = 0; c < ncls; c++) {
        int ph = c / s, pw = c - ph * s;
        int ihf = ((ph - g.pad) % s + s) % s, iwf = ((pw - g.pad) % s + s) % s;
        int padl_h = (TH - 1) - (ihf + g.pad - ph) / s, padl_w = (TW - 1) - (iwf + g.pad - pw) / s;
        int Hc = Hin / s, Wc = Win / s;
        int up_h = Hc - g.Ho - padl_h, up_w = Wc - g.Wo - padl_w;
        if (int rc = encode_act_map(&p.cls[c].amap, dy, (long)g.G * g.B, g.Ho, g.Wo, g.Cout, -padl_w, -padl_h, up_w, up_h, 1, p.bk)) return rc;
        p.cls[c].w0 = -padl_w; p.cls[c].h0 = -padl_h;
        p.cls[c].out_h0 = ihf; p.cls[c].out_w0 = iwf;
        p.cls[c].wrow_off = c * CinP;
    }
    p.ncls = ncls;
    p.G = g.G; p.xg_images = g.B;
    p.B = g.B; p.P = Hin / s; p.Q = Win / s;
    p.Cin = g.Cout; p.Cout = g.Cin; p.KH = TH; p.KW = TW; p.stride = 1;
    p.out_H = Hin; p.out_W = Win; p.out_sh = s; p.out_sw = s;
    p.w_rows_per_group = ncls * CinP;
    p.y = d_seen; p.bias = nullptr;
    p.addend = g.ups ? nullptr : addend; p.mask_src = g.ups ? nullptr : mask_src;
    p.act = CG_ACT_NONE; p.slope = mask_slope;
    if (int rc = launch_tc(p, st)) return rc;
    if (g.ups) return pool2x2_sum(d_seen, dx, addend, mask_src, mask_slope, (long)g.G * g.B, g.H, g.W, g.Cin, st);
    return CG_OK;
}


// ------------------------------------------------------------------------------------------------
// weight gradient on tensor cores
//
//   dW[g][co][kh][kw][ci] = sum over pixels m of dy[g][m][co] * x[g][n][p*s-pad+kh][q*s-pad+kw][ci]
//
// GEMM per (group, BM-cout tile, filter tap, BN-ci tile, pixel split):  D[BM co][BN ci] += dy^T[co][pixels] * x[pixels][ci],
// the reduction (K) dimension being pixels.  In the channels-last tensors both operands are contiguous along their M / N
// dimension (MN-major), and wgmma takes TF32 operands K-major only, so every 32-pixel chunk goes through a transform stage:
// all threads load it from global memory (coalesced float4 along the channels, zero outside the image and past the split) into
// registers and store it transposed and TF32-rounded into the K-major 128-byte-swizzled layout the forward kernel's TMA
// produces.  Each warpgroup then multiplies 64 output channels of the chunk by the whole BN tile with wgmma.  Two shared-memory
// buffers: the global loads and the transposed stores of chunk c+1 overlap the MMAs of chunk c.  Splits of the pixel range
// write partial results that a second kernel sums in a fixed order (deterministic).
// ------------------------------------------------------------------------------------------------
constexpr int WG_BK = 32;       // pixels per chunk = one 128-byte K-major row

struct WgParams {
    const float* x; const float* dy; float* out;
    int G, xg_images, B, H, W, Ho, Wo, Cin, Cout, KH, KW, stride, pad;
    long Mpix, chunk;
    int ci_tiles;
};

__device__ __forceinline__ float f4_at(const float4& v, int j) { return j == 0 ? v.x : j == 1 ? v.y : j == 2 ? v.z : v.w; }

// rows r0..r0+3 of a K-major 128-byte-swizzled operand tile (rows of 32 fp32), column k
__device__ __forceinline__ void store_kmajor4(uint8_t* tile, int r0, int k, const float4& v) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int r = r0 + j;
        *reinterpret_cast<float*>(tile + (r >> 3) * 1024 + (r & 7) * 128 + (((k >> 2) ^ (r & 7)) << 4) + (k & 3) * 4) = to_tf32(f4_at(v, j));
    }
}

template <int BM, int BN>
__global__ void __launch_bounds__(2 * BM) wgrad_tc_kernel(const __grid_constant__ WgParams p) {
    constexpr int NWARPS = 2 * BM / 32;             // BM / 64 warpgroups
    constexpr int NA = 4, NB = 4 * BN / BM;         // float4 loads per thread and chunk: dy, x
    constexpr int A_BYTES = BM * 128, STAGE = (BM + BN) * 128;
    pdl_trigger();
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int lane = threadIdx.x & 31;
    const int warp = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 5, 0);  // warp-uniform for the compiler
    const int wg = warp >> 2;
    const int tap = blockIdx.x / p.ci_tiles, ci0 = (blockIdx.x % p.ci_tiles) * BN;
    const int kh = tap / p.KW, kw = tap - kh * p.KW;
    const int co0 = blockIdx.y * BM;
    const int g = blockIdx.z % p.G, split = blockIdx.z / p.G;
    const long m_begin = (long)split * p.chunk;
    long m_end = m_begin + p.chunk;
    if (m_end > p.Mpix) m_end = p.Mpix;
    const int PQ = p.Ho * p.Wo;
    const float* dyg = p.dy + (long)g * p.Mpix * p.Cout;
    // loader mapping: a warp covers 8 pixels x 4 float4 columns per load (full 64-byte runs in global memory, at most 2-way bank
    // conflicts on the transposed stores); load i of warp w reads column block (w + NWARPS i) / 4 of this thread's single pixel
    const int kq = lane & 7, cq = lane >> 3;
    const int k_own = 8 * (warp & 3) + kq;
    pdl_wait();

    float4 ra[NA], rb[NB];
    auto gload = [&](long m0) {
        const long m = m0 + k_own;
        const bool in = m < m_end;
        const float* xs = nullptr;
        if (in) {
            const int img = (int)(m / PQ);
            const int rem = (int)(m - (long)img * PQ);
            const int oh = rem / p.Wo, ow = rem - oh * p.Wo;
            const int ih = oh * p.stride - p.pad + kh, iw = ow * p.stride - p.pad + kw;
            if (ih >= 0 && ih < p.H && iw >= 0 && iw < p.W) xs = p.x + (((long)(g * p.xg_images + img) * p.H + ih) * p.W + iw) * p.Cin;
        }
#pragma unroll
        for (int i = 0; i < NA; i++) {
            const int co = co0 + 4 * (4 * ((warp + NWARPS * i) >> 2) + cq);
            ra[i] = in && co < p.Cout ? __ldg(reinterpret_cast<const float4*>(dyg + m * p.Cout + co)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int i = 0; i < NB; i++) {
            const int ci = ci0 + 4 * (4 * ((warp + NWARPS * i) >> 2) + cq);
            rb[i] = xs && ci < p.Cin ? __ldg(reinterpret_cast<const float4*>(xs + ci)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    auto sstore = [&](int buf) {
        uint8_t* sa = smem + buf * STAGE;
#pragma unroll
        for (int i = 0; i < NA; i++) store_kmajor4(sa, 4 * (4 * ((warp + NWARPS * i) >> 2) + cq), k_own, ra[i]);
#pragma unroll
        for (int i = 0; i < NB; i++) store_kmajor4(sa + A_BYTES, 4 * (4 * ((warp + NWARPS * i) >> 2) + cq), k_own, rb[i]);
    };

    const uint64_t desc0 = make_kmajor_sw128_desc(0);
    const long nchunks = (m_end - m_begin + WG_BK - 1) / WG_BK;
    float acc[BN / 2];
    gload(m_begin);
    sstore(0);
    fence_proxy_async();
    __syncthreads();
    for (long c = 0; c < nchunks; c++) {
        const int buf = (int)(c & 1);
        if (c + 1 < nchunks) gload(m_begin + (c + 1) * WG_BK);
        const uint32_t sa = smem_u32(smem + buf * STAGE) + wg * (64 * 128);
        const uint32_t sb = smem_u32(smem + buf * STAGE) + A_BYTES;
        const uint64_t adesc = desc0 | (uint64_t)((sa & 0x3FFFF) >> 4), bdesc = desc0 | (uint64_t)((sb & 0x3FFFF) >> 4);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < WG_BK / 8; kk++)  // 8 tf32 (32 bytes) along K per step: +2 in the address field
            wgmma_tf32<BN>(acc, adesc + (uint64_t)(kk * 2), bdesc + (uint64_t)(kk * 2), (c | kk) != 0 ? 1 : 0);
        wgmma_commit();
        if (c + 1 < nchunks) {
            wgmma_wait<1>();  // this warpgroup's MMAs of chunk c-1 have retired ...
            __syncthreads();  // ... and the other warpgroup's: the other buffer is free
            sstore(buf ^ 1);
            fence_proxy_async();
            __syncthreads();
        }
    }
    wgmma_wait<0>();
    wgmma_reg_fence(acc, BN / 2);

    const long Ktot = (long)p.KH * p.KW * p.Cin;
    float* out = p.out + (long)split * p.G * p.Cout * Ktot;
    const int row0 = co0 + wg * 64 + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
        const int ci = ci0 + 8 * j + 2 * (lane & 3);
        if (ci >= p.Cin) continue;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int co = row0 + 8 * h;
            if (co < p.Cout)
                *reinterpret_cast<float2*>(out + ((long)g * p.Cout + co) * Ktot + (long)tap * p.Cin + ci) =
                    make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
    }
}

__global__ void reduce_splits_tc_kernel(const float* __restrict__ part, float* __restrict__ out, long n4, int splits) {
    pdl_trigger();
    pdl_wait();
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n4) return;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k = 0; k < splits; k++) {
        float4 v = __ldg(reinterpret_cast<const float4*>(part) + (long)k * n4 + i);
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    reinterpret_cast<float4*>(out)[i] = s;
}

// Tile shape: 128 output / input channels where the layer has more than 64, else 64
static int wg_bm(const cg_conv_geom& g) { return g.Cout > 64 ? 128 : 64; }
static int wg_bn(const cg_conv_geom& g) { return g.Cin > 64 ? 128 : 64; }

// Split the pixel range until the launch fills every SM several times over (up to 3 co-resident CTAs each), keeping >= 8 chunks
// of work per split and the partial sums <= 64 MB.
static void wg_plan(const cg_conv_geom& g, int& splits, long& chunk) {
    const long Mpix = (long)g.B * g.Ho * g.Wo;
    const long base = (long)g.G * cdiv(g.Cout, wg_bm(g)) * cdiv(g.Cin, wg_bn(g)) * g.KH * g.KW;
    const long target = 3L * sm_count_now();
    long s = (target + base - 1) / base;
    long maxs = Mpix / (8 * WG_BK);
    const long out_bytes = (long)g.G * g.Cout * g.KH * g.KW * g.Cin * 4;
    const long cap = (64l << 20) / (out_bytes > 0 ? out_bytes : 1);
    if (maxs > cap) maxs = cap;
    if (maxs > 64) maxs = 64;
    if (s > maxs) s = maxs;
    if (s < 1) s = 1;
    chunk = ((Mpix + s - 1) / s + WG_BK - 1) / WG_BK * WG_BK;
    splits = (int)((Mpix + chunk - 1) / chunk);
}

// ------------------------------------------------------------------------------------------------
// weight gradient of stride-1 and stride-2 convolutions with KH*KW > 1: TMA-fed wgmma pipeline, shifted operand from registers
//
// For tap k = (kh, kw) and stride s,  dW[k][co][ci] = sum over dy pixels o of x[s o + k - pad][ci] * dy[o][co],
// out-of-range x pixels counting as zero.  The reduction (K) runs over dy pixels, x is read at tap-shifted pixels.
// * Writing k - pad = s a + r with 0 <= r < s (per axis), x row s oh + k - pad is row oh + a of the row-parity-r sub-grid of x:
//   in a parity view of x every tap is a whole-pixel shift a of the dy grid.  The view is a 5-D tiled map over the unchanged
//   channels-last memory, (s Cin, W / s, s, H / s, N): the column parity is folded into the channel coordinate (r_w Cin + ci), the
//   row parity is its own coordinate.  For s = 1 it is the plain (C, W, 1, H, N) view.
// * dy is "copied": a transpose kernel writes it channel-major [img][Cout][Ho][Wo], TF32-rounded, into the workspace once per
//   call, and a 4-D tiled map with a (32 px, 1, BN channels, 1) box brings 32 pixels straight into the K-major
//   128-byte-swizzled layout wgmma reads as its B operand.  Where Wo >= 32 the map is (Wo, Ho, C, N) and a chunk is 32 pixels of
//   one row; chunk starts are multiples of 32 pixels, so the innermost TMA coordinate stays aligned, and a partial last chunk of
//   a row is zero-filled.  Where Wo < 32 divides 32 (and 32 divides Ho Wo) a chunk is 32 / Wo whole rows, and the same memory
//   is mapped as (32, Ho Wo / 32, C, N).
// * x ("direct") is read through the parity view, box (32 channels, 32 px, 1, 1, 1), or (32 channels, Wo px, 1, 32 / Wo rows, 1)
//   for whole-row chunks; both land as [pixel][32 channels] in the chunk's pixel order.  The tap shift moves the W / s and H / s
//   coordinates, which are outer dimensions, so starts off the map are legal and zero-filled (the padding).
//   That tile is MN-major, which wgmma cannot take as a TF32 shared-memory operand; the consumers read their A fragments out of
//   it with LDS, round them to TF32 and issue the register-A ("RS") form of wgmma.
// * M = Cin, N = Cout: the epilogue stores D transposed into dw[g][co][kh][kw][ci].
// * Same arithmetic as wgrad_tc_kernel: the same TF32-rounded operands, the same pixel splits (wg_plan), and within a split the
//   same 8-pixel k-steps in the same order, so where a 32-pixel chunk is 32 consecutive pixels of dy (Wo % 32 == 0, or whole-row
//   chunks) both kernels produce the same bits.  Training amplifies any rounding difference in the weight gradients within a
//   few steps, so a kernel that merely agreed to rounding would change what a training run computes.
// * Warp-specialised persistent CTAs as in conv_tc_kernel: one TMA producer thread, BM / 64 consumer warpgroups, a full / empty
//   mbarrier ring.  Work units (pixel split, group, tap, M tile, N tile) are walked split-major, so that the CTAs running at the
//   same time read the same pixel range and the KH*KW re-reads of it come from L2.  Splits write partials that
//   reduce_splits_tc_kernel sums in a fixed order (deterministic).
// ------------------------------------------------------------------------------------------------
thread_local int g_wgrad_tma = 1;  // mode bit 25 clears it: every layer this kernel serves stays on wgrad_tc_kernel

constexpr int WT_MAX_STAGES = 8;

struct WtParams {
    CUtensorMap amap;               // parity view of x, channels-last
    CUtensorMap bmap;               // channel-major copy of dy
    float* out;                     // [split][G][Cout][KH][KW][Cin]
    int G, KW, taps, M, N, Cin, Cout;
    int a_gimg, b_gimg;             // images per group in the x / dy-copy map (0: input shared by the council)
    int Hc, cpr, rows;              // per image: chunk rows, 32-pixel chunks per chunk row; dy rows per chunk row
    int pad, s_log2;                // x pixel = stride * dy pixel + tap - pad, stride = 1 << s_log2
    long chunks, split_chunks;      // chunks per member, per split
    int units, stages;
};

// Accumulator row r (0..15) of warp w of a consumer warpgroup <-> channel of the direct tile.  With the 128-byte swizzle, channel c of
// pixel k sits in 16-byte chunk (c / 4) ^ (k % 8) of the pixel's 128-byte row.  One A-fragment LDS of a warp reads 8 rows at 4
// consecutive pixels (k % 8 in 0..3 or 4..7); if the 8 rows were 8 consecutive channels they would span 2 chunks, and
// XOR-ed with 4 pixel values those give only 4 distinct chunks: 2-way bank conflicts.  Rows r = 0..3 -> channels c..c+3 and
// r = 4..7 -> c+16..c+19 instead come from chunks q and q + 4 (q even), which the XOR keeps apart: 8 chunks, 32 banks.
// Rows 8..15 take the channels 4 above those of rows 0..7; warps w and w^1 share one 32-channel box.
// shared-memory load of one A fragment element, rounded to TF32 (the tensor core would truncate it)
__device__ __forceinline__ uint32_t lds_tf32(uint32_t addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return tf32_bits(v);
}
__device__ __forceinline__ int wt_row_channel(int w, int r) { return 32 * (w >> 1) + 8 * (w & 1) + (r & 3) + 16 * ((r >> 2) & 1) + 4 * (r >> 3); }

template <int BM, int BN>
__global__ void __launch_bounds__(2 * BM + 128, BM == 64 ? 2 : 1) wgrad_tma_kernel(const __grid_constant__ WtParams p) {
    constexpr int A_BOX = 32 * 128;                // 32 channels x 32 pixels
    constexpr int STAGE = (BM + BN) * 128;         // [A box 0 .. BM/32-1][B: BN rows of 32 pixels]
    constexpr int NCW = BM / 64;                   // consumer warpgroups
    pdl_trigger();
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0), tid = threadIdx.x & 127;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * STAGE);
    uint64_t* empty_bar = full_bar + p.stages;
    const int MT = (p.M + BM - 1) / BM, NT = (p.N + BN - 1) / BN;

    if (threadIdx.x == 0) {
        prefetch_tmap(&p.amap);
        prefetch_tmap(&p.bmap);
        for (int s = 0; s < p.stages; s++) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], NCW);
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();

    if (wg == 0) {
        // ===================== TMA producer =====================
        if (tid == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
                int r = u / NT;
                const int n0 = (u - r * NT) * BN;
                const int m0 = (r % MT) * BM;
                r /= MT;
                const int tap = r % p.taps;
                r /= p.taps;
                const int g = r % p.G, split = r / p.G;
                const int kh = tap / p.KW, kw = tap - kh * p.KW;
                // tap offset = stride * a + r per axis, 0 <= r < stride (arithmetic shift: floor division by a power of two)
                const int ah = (kh - p.pad) >> p.s_log2, rh = kh - p.pad - (ah << p.s_log2);
                const int aw = (kw - p.pad) >> p.s_log2, rw = kw - p.pad - (aw << p.s_log2);
                int nbox = (p.M - m0) / 32;                // whole 32-channel boxes inside the tensor (M % 32 == 0)
                if (nbox > BM / 32) nbox = BM / 32;       // rows past M are never stored: their boxes are not loaded
                const uint32_t tx = (uint32_t)(nbox * A_BOX + BN * 128);
                long c = split * p.split_chunks, c_end = c + p.split_chunks;
                if (c_end > p.chunks) c_end = p.chunks;
                const long per_img = (long)p.Hc * p.cpr;
                int img = (int)(c / per_img);
                int rem = (int)(c - img * per_img);
                int h = rem / p.cpr, wq = rem - h * p.cpr;
                for (; c < c_end; c++) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    uint8_t* sa = smem + (size_t)stage * STAGE;
                    mbar_expect_tx(&full_bar[stage], tx);
                    const int w0 = wq * 32;
                    for (int j = 0; j < nbox; j++)
                        tma_load_5d(&p.amap, &full_bar[stage], sa + j * A_BOX, rw * p.Cin + m0 + 32 * j, w0 + aw, rh, h * p.rows + ah,
                                    g * p.a_gimg + img);
                    tma_load_4d(&p.bmap, &full_bar[stage], sa + BM * 128, w0, h, n0, g * p.b_gimg + img);
                    if (++wq == p.cpr) { wq = 0; if (++h == p.Hc) { h = 0; ++img; } }
                    if (++stage == p.stages) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ===================== MMA + epilogue (consumer warpgroups) =====================
    const int cw = wg - 1, warp4 = tid >> 5, lane = tid & 31;
    const int wl = 2 * cw + (warp4 >> 1);                      // this warp's 32-channel box ...
    const int wsub = warp4 & 1;                                // ... and which half of it (see wt_row_channel)
    const int ch0 = wt_row_channel(wsub, lane >> 2);            // channel in the box of accumulator row lane / 4; row + 8: ch0 + 4
    const int kq = lane & 3;
    // byte offsets of a[0..3] in the box for k-step 0: (ch0, kq), (ch0 + 4, kq), (ch0, kq + 4), (ch0 + 4, kq + 4); k-step kk adds 1024 kk
    auto swz = [](int ch, int k) { return k * 128 + ((((ch >> 2) ^ (k & 7))) << 4) + (ch & 3) * 4; };
    const int off0 = swz(ch0, kq) + wl * A_BOX, off1 = swz(ch0 + 4, kq) + wl * A_BOX;
    const int off2 = swz(ch0, kq + 4) + wl * A_BOX, off3 = swz(ch0 + 4, kq + 4) + wl * A_BOX;
    const uint64_t desc0 = make_kmajor_sw128_desc(0);
    const long Ktot = (long)p.taps * p.Cin;
    float acc[BN / 2];
    uint32_t af[2][4];
    int stage = 0;
    uint32_t phase = 0;
    for (int u = blockIdx.x; u < p.units; u += gridDim.x) {
        int r = u / NT;
        const int n0 = (u - r * NT) * BN;
        const int m0 = (r % MT) * BM;
        r /= MT;
        const int tap = r % p.taps;
        r /= p.taps;
        const int g = r % p.G, split = r / p.G;
        long c0 = split * p.split_chunks, c_end = c0 + p.split_chunks;
        if (c_end > p.chunks) c_end = p.chunks;
        int prev = -1;
        for (long c = c0; c < c_end; c++) {
            mbar_wait(&full_bar[stage], phase);
            const uint32_t sa32 = smem_u32(smem + (size_t)stage * STAGE);
            const uint32_t sb = sa32 + BM * 128;
            const uint64_t bdesc = desc0 | (uint64_t)((sb & 0x3FFFF) >> 4);
#pragma unroll
            for (int kk = 0; kk < 4; kk++) {
                // double-buffered fragments: af[kk & 1] was last read by the MMA of k-step kk - 2, which the wait below retired
                uint32_t* a = af[kk & 1];
                a[0] = lds_tf32(sa32 + off0 + 1024 * kk);
                a[1] = lds_tf32(sa32 + off1 + 1024 * kk);
                a[2] = lds_tf32(sa32 + off2 + 1024 * kk);
                a[3] = lds_tf32(sa32 + off3 + 1024 * kk);
                wgmma_fence();  // orders the fragment writes above (and the accumulators) before the asynchronous MMA reads them
                wgmma_tf32_rs<BN>(acc, a, bdesc + (uint64_t)(kk * 2), (c != c0 || kk) ? 1 : 0);
                wgmma_commit();
                wgmma_wait<1>();  // the MMA of k-step kk - 1 has retired: its fragment buffer is free
                // at k-step 0 that was the last MMA of the previous chunk: its stage can be refilled
                if (kk == 0 && prev >= 0 && tid == 0) mbar_arrive(&empty_bar[prev]);
            }
            prev = stage;
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_reg_fence(acc, BN / 2);
        if (tid == 0) mbar_arrive(&empty_bar[prev]);

        float* out = p.out + ((long)split * p.G + g) * p.Cout * Ktot + (long)tap * p.Cin;
        const int cq = 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int m = m0 + 32 * wl + ch0 + 4 * h;
            if (m >= p.M) continue;
#pragma unroll
            for (int j = 0; j < BN / 8; j++) {
                const int n = n0 + 8 * j + cq;
                if (n >= p.N) break;
                const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                out[(long)n * Ktot + m] = v0;  // m = ci, n = co
                out[(long)(n + 1) * Ktot + m] = v1;
            }
        }
    }
}

// [img][H][W][C] -> [img][C][H][W], rounded to TF32 as wgrad_tc_kernel rounds its operands: 32 pixels x 32 channels per block
// through a padded shared tile; float4 reads along C, 128-byte writes along W.  grid (W tiles * C tiles, H, images)
__global__ void __launch_bounds__(256) nhwc_to_nchw_tf32_kernel(const float* __restrict__ src, float* __restrict__ dst, int H, int W, int C) {
    pdl_trigger();
    pdl_wait();
    __shared__ float tile[32][33];
    const int ct = C / 32;
    const int w0 = (blockIdx.x / ct) * 32, c0 = (blockIdx.x % ct) * 32;
    const int h = blockIdx.y;
    const long img = blockIdx.z;
    const int t = threadIdx.x;
    const int px = t >> 3, c4 = (t & 7) * 4;
    if (w0 + px < W) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(src + ((img * H + h) * W + w0 + px) * C + c0 + c4));
        tile[c4][px] = v.x; tile[c4 + 1][px] = v.y; tile[c4 + 2][px] = v.z; tile[c4 + 3][px] = v.w;
    }
    __syncthreads();
    const int tx = t & 31, ty = t >> 5;
    if (w0 + tx >= W) return;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int c = ty + 8 * j;
        dst[((img * C + c0 + c) * H + h) * W + w0 + tx] = to_tf32(tile[c][tx]);
    }
}

// dy rows per 32-pixel chunk: 32 / Wo whole rows where Wo < 32 divides 32 and the chunks tile each image, else 1
static int wt_rows(const cg_conv_geom& g) { return g.Wo < 32 && 32 % g.Wo == 0 && g.Ho * g.Wo % 32 == 0 ? 32 / g.Wo : 1; }

bool tc_wgrad_tma_supported(const cg_conv_geom& g) {
    if (!g_wgrad_tma || g.ups || g.KH * g.KW <= 1) return false;
    if (g.stride != 1 && g.stride != 2) return false;
    if (g.H % g.stride || g.W % g.stride) return false;  // the parity view of x is made of whole stride x stride cells
    if (g.Cin % 32 != 0 || g.Cout % 32 != 0) return false;
    init_driver();
    if (!g_encode_tiled) return false;
    if ((long)g.B * g.Ho * g.Wo < 256) return false;
    const int rows = wt_rows(g), Hs = g.H / g.stride, Ws = g.W / g.stride;  // x box: 32 pixels of one row, or `rows` rows of Wo
    if (rows > 1) return Ws >= g.Wo && Hs >= rows;
    return Ws >= 32 && g.Wo >= 32 && g.Wo % 4 == 0;  // Wo % 4: TMA strides of the copy are multiples of 16 bytes
}

struct WtPlan {
    int bm, bn, rows, cpr, splits, slots;
    long chunks, split_chunks, copy_bytes, part_bytes;
};

static WtPlan wt_plan(const cg_conv_geom& g) {
    WtPlan q;
    // one consumer warpgroup (BM = 64) where Cin <= 64; 64 x 128 tiles there read each x chunk once for 128 output channels,
    // 1.5x the rate of 64 x 64 tiles on the 4x4 64->128 layers
    q.bm = g.Cin > 64 ? 128 : 64;
    q.bn = q.bm == 128 && g.Cout >= 256 ? 256 : g.Cout > 64 ? 128 : 64;
    q.rows = wt_rows(g);
    q.cpr = q.rows > 1 ? 1 : cdiv(g.Wo, 32);
    q.chunks = (long)g.B * (g.Ho / q.rows) * q.cpr;
    q.copy_bytes = (((long)g.G * g.B * g.Ho * g.Wo * g.Cout * 4) + 1023) & ~1023L;
    q.slots = (q.bm == 64 ? 2 : 1) * sm_count_now();  // two CTAs per SM for the single-warpgroup tiles
    // the pixel splits of wgrad_tc_kernel (see the section comment); `chunk` is a multiple of 32 pixels
    int splits;
    long chunk;
    wg_plan(g, splits, chunk);
    q.split_chunks = g.Wo % 32 == 0 || q.rows > 1 ? chunk / 32 : (q.chunks + splits - 1) / splits;
    q.splits = (int)((q.chunks + q.split_chunks - 1) / q.split_chunks);
    q.part_bytes = q.splits > 1 ? (long)q.splits * g.G * g.Cout * g.KH * g.KW * g.Cin * 4 : 0;
    return q;
}

template <int BM, int BN>
static int launch_wt(WtParams& p, int slots, cudaStream_t st) {
    constexpr int STAGE = (BM + BN) * 128;
    // BM = 64: two CTAs per SM (228 KB of shared memory per SM, 1 KB of it reserved per CTA)
    int stages = ((BM == 64 ? 110 : 225) * 1024 - 1024 - 2 * WT_MAX_STAGES * 8) / STAGE;
    if (stages > WT_MAX_STAGES) stages = WT_MAX_STAGES;
    p.stages = stages;
    const size_t smem = (size_t)stages * STAGE + 1024 + 2 * stages * 8;
    static PerDeviceOnce attr_set;
    if (attr_set.first()) {
        cudaError_t e = cudaFuncSetAttribute(wgrad_tma_kernel<BM, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) {
            attr_set.reset();
            set_error("cudaFuncSetAttribute(wgrad_tma_kernel): %s", cudaGetErrorString(e));
            return CG_ERR_CUDA;
        }
    }
    const int grid = p.units < slots ? p.units : slots;
    launch_k(wgrad_tma_kernel<BM, BN>, grid, 2 * BM + 128, smem, st, p);
    return check_launch("wgrad_tma_kernel");
}

static int tc_conv_wgrad_tma(const cg_conv_geom& g, const float* x, const float* dy, float* dw, void* ws, cudaStream_t st) {
    const WtPlan q = wt_plan(g);
    float* copy = (float*)ws;
    float* part = (float*)((uint8_t*)ws + q.copy_bytes);
    const long nimg_x = g.x_groups == 1 ? g.B : (long)g.G * g.B, nimg_dy = (long)g.G * g.B;
    launch_k(nhwc_to_nchw_tf32_kernel, dim3(cdiv(g.Wo, 32) * (g.Cout / 32), g.Ho, (unsigned)nimg_dy), 256, 0, st, dy, copy, g.Ho, g.Wo,
             g.Cout);
    if (int rc = check_launch("nhwc_to_nchw_tf32")) return rc;

    // Both maps move raw fp32 (the copy is already rounded, x is rounded in registers), whatever a TF32 map would do to the low bits.
    WtParams p{};
    // x: parity view (s C, W / s, s, H / s, N) of the channels-last tensor, box (32 channels, 32 px, 1, 1, 1) or
    // (32 channels, Wo px, 1, rows, 1)
    {
        const int s = g.stride, box_w = q.rows > 1 ? g.Wo : 32;
        MapKey k{};
        k.ptr = x; k.a = nimg_x; k.b = ((int64_t)g.H << 32) | (uint32_t)g.W;
        k.v[0] = g.Cin; k.v[1] = s; k.v[2] = box_w; k.v[3] = q.rows; k.v[7] = 3;
        int rc = cached_map(&p.amap, k, [&](CUtensorMap* m) {
            cuuint64_t dims[5] = {(cuuint64_t)s * g.Cin, (cuuint64_t)(g.W / s), (cuuint64_t)s, (cuuint64_t)(g.H / s), (cuuint64_t)nimg_x};
            cuuint64_t strides[4] = {(cuuint64_t)s * g.Cin * 4, (cuuint64_t)g.W * g.Cin * 4, (cuuint64_t)s * g.W * g.Cin * 4,
                                     (cuuint64_t)g.H * g.W * g.Cin * 4};
            cuuint32_t box[5] = {32, (cuuint32_t)box_w, 1, (cuuint32_t)q.rows, 1}, estr[5] = {1, 1, 1, 1, 1};
            CUresult r = g_encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, (void*)x, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) {
                set_error("cuTensorMapEncodeTiled(wgrad x N=%ld H=%d W=%d C=%d stride %d box %dx%d) failed: %d", nimg_x, g.H, g.W, g.Cin, s,
                          q.rows, box_w, (int)r);
                return (int)CG_ERR_CUDA;
            }
            return (int)CG_OK;
        });
        if (rc) return rc;
    }
    // channel-major copy of dy: (Wo, Ho, C, N), or (32, Ho Wo / 32, C, N) for whole-row chunks; box (32 px, 1, BN channels, 1)
    {
        const int cw = q.rows > 1 ? 32 : g.Wo;
        MapKey k{};
        k.ptr = copy; k.a = nimg_dy; k.b = ((int64_t)g.Ho << 32) | (uint32_t)g.Wo; k.v[0] = g.Cout; k.v[1] = q.bn; k.v[7] = 4;
        int rc = cached_map(&p.bmap, k, [&](CUtensorMap* m) {
            cuuint64_t dims[4] = {(cuuint64_t)cw, (cuuint64_t)g.Ho * g.Wo / cw, (cuuint64_t)g.Cout, (cuuint64_t)nimg_dy};
            cuuint64_t strides[3] = {(cuuint64_t)cw * 4, (cuuint64_t)g.Ho * g.Wo * 4, (cuuint64_t)g.Cout * g.Ho * g.Wo * 4};
            cuuint32_t box[4] = {32, 1, (cuuint32_t)q.bn, 1}, estr[4] = {1, 1, 1, 1};
            CUresult r = g_encode_tiled(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)copy, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            if (r != CUDA_SUCCESS) {
                set_error("cuTensorMapEncodeTiled(wgrad dy copy N=%ld H=%d W=%d C=%d) failed: %d", nimg_dy, g.Ho, g.Wo, g.Cout, (int)r);
                return (int)CG_ERR_CUDA;
            }
            return (int)CG_OK;
        });
        if (rc) return rc;
    }
    p.out = q.splits == 1 ? dw : part;
    p.G = g.G; p.KW = g.KW; p.taps = g.KH * g.KW; p.M = g.Cin; p.N = g.Cout; p.Cin = g.Cin; p.Cout = g.Cout;
    p.a_gimg = g.x_groups == 1 ? 0 : g.B;
    p.b_gimg = g.B;
    p.Hc = g.Ho / q.rows; p.cpr = q.cpr; p.rows = q.rows;
    p.pad = g.pad; p.s_log2 = g.stride == 2;
    p.chunks = q.chunks; p.split_chunks = q.split_chunks;
    p.units = q.splits * g.G * p.taps * cdiv(g.Cin, q.bm) * cdiv(g.Cout, q.bn);
    int rc;
    if (q.bm == 64) rc = q.bn == 64 ? launch_wt<64, 64>(p, q.slots, st) : launch_wt<64, 128>(p, q.slots, st);
    else if (q.bn == 64) rc = launch_wt<128, 64>(p, q.slots, st);
    else if (q.bn == 128) rc = launch_wt<128, 128>(p, q.slots, st);
    else rc = launch_wt<128, 256>(p, q.slots, st);
    if (rc) return rc;
    if (q.splits > 1) {
        long n4 = (long)g.G * g.Cout * g.KH * g.KW * g.Cin / 4;
        launch_k(reduce_splits_tc_kernel, cdiv(n4, 256), 256, 0, st, (const float*)part, dw, n4, q.splits);
        return check_launch("reduce_splits_tc");
    }
    return CG_OK;
}

bool tc_wgrad_supported(const cg_conv_geom& g) {
    if (tc_wgrad_tma_supported(g)) return true;
    if (g.ups) return false;
    if (g.Cin % 32 != 0 || g.Cout % 4 != 0) return false;
    long Mpix = (long)g.B * g.Ho * g.Wo;
    return Mpix % WG_BK == 0 && Mpix >= 256;
}

size_t tc_wgrad_ws(const cg_conv_geom& g) {
    if (tc_wgrad_tma_supported(g)) {
        const WtPlan q = wt_plan(g);
        return (size_t)(q.copy_bytes + q.part_bytes);
    }
    int splits; long chunk;
    wg_plan(g, splits, chunk);
    if (splits == 1) return 0;
    return (size_t)splits * g.G * g.Cout * g.KH * g.KW * g.Cin * sizeof(float);
}

int tc_sm_count() { return sm_count_now(); }

int tc_conv_wgrad(const cg_conv_geom& g, const float* x, const float* dy, float* dw, void* ws, size_t ws_bytes, cudaStream_t st) {
    if (tc_wgrad_tma_supported(g)) {
        size_t need = tc_wgrad_ws(g);
        if (need > ws_bytes) {
            set_error("conv_wgrad(tc, tma): workspace %zu < %zu bytes", ws_bytes, need);
            return CG_ERR_WORKSPACE;
        }
        return tc_conv_wgrad_tma(g, x, dy, dw, ws, st);
    }
    WgParams p{};
    int splits;
    wg_plan(g, splits, p.chunk);
    size_t need = tc_wgrad_ws(g);
    if (need > ws_bytes) {
        set_error("conv_wgrad(tc): workspace %zu < %zu bytes", ws_bytes, need);
        return CG_ERR_WORKSPACE;
    }
    p.x = x; p.dy = dy; p.out = splits == 1 ? dw : (float*)ws;
    p.G = g.G; p.xg_images = g.x_groups == 1 ? 0 : g.B;
    p.B = g.B; p.H = g.H; p.W = g.W; p.Ho = g.Ho; p.Wo = g.Wo; p.Cin = g.Cin; p.Cout = g.Cout;
    p.KH = g.KH; p.KW = g.KW; p.stride = g.stride; p.pad = g.pad;
    p.Mpix = (long)g.B * g.Ho * g.Wo;
    const int bm = wg_bm(g), bn = wg_bn(g);
    p.ci_tiles = cdiv(g.Cin, bn);
    void (*kern)(WgParams) = bm == 128 ? (bn == 128 ? wgrad_tc_kernel<128, 128> : wgrad_tc_kernel<128, 64>)
                                       : (bn == 128 ? wgrad_tc_kernel<64, 128> : wgrad_tc_kernel<64, 64>);
    const size_t smem = 2 * (size_t)(bm + bn) * 128 + 1024;
    static PerDeviceOnce attr_set;
    if (attr_set.first()) {
        void (*all[4])(WgParams) = {wgrad_tc_kernel<128, 128>, wgrad_tc_kernel<128, 64>, wgrad_tc_kernel<64, 128>, wgrad_tc_kernel<64, 64>};
        for (auto k : all) {
            cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 256 * 128 + 1024);
            if (e != cudaSuccess) {
                attr_set.reset();
                set_error("cudaFuncSetAttribute(wgrad_tc_kernel): %s", cudaGetErrorString(e));
                return CG_ERR_CUDA;
            }
        }
    }
    launch_k(kern, dim3(p.ci_tiles * g.KH * g.KW, cdiv(g.Cout, bm), g.G * splits), 2 * bm, smem, st, p);
    if (int rc = check_launch("wgrad_tc_kernel")) return rc;
    if (splits > 1) {
        long n4 = (long)g.G * g.Cout * g.KH * g.KW * g.Cin / 4;
        launch_k(reduce_splits_tc_kernel, cdiv(n4, 256), 256, 0, st, (const float*)ws, dw, n4, splits);
        return check_launch("reduce_splits_tc");
    }
    return CG_OK;
}

}  // namespace cg
