// wgmma tensor-core GEMM for sm_90a:  C = act(alpha * A * B^T + bias) + residual  on SB16 operands.
//
// Error-compensated bf16x3: every float32 operand value travels as hi + lo bfloat16 planes and each
// k-step issues three wgmmas into the same register accumulator:  A_hi*B_hi + A_lo*B_hi + A_hi*B_lo
// (the dropped lo*lo term is ~2^-16 relative).  That keeps logits and cross-attention scores within
// the 1e-3 bar of the reference's float32 CPU path while running on the tensor cores.
//
// Both kernels feed 128-column output tiles from an operand ring: per k-block the TMA producer lane loads 4 boxes
// (A_hi, A_lo, B_hi, B_lo; 64 bf16 wide, SWIZZLE_128B) into one ring stage; full[s] completes on the byte count,
// empty[s] once the consumer warps have retired the k-block's wgmmas.  Batched problems (two batch levels) are extra
// tensor-map dimensions; M/N/K tails rely on TMA zero fill.  Every output element sums the same k-blocks, k16 steps and
// terms (hi*hi, lo*hi, hi*lo) in the same order in every kernel here, so they give bit-identical results.
//
// gemm_tc_kernel (encoder, cross-K/V, prefill: more than one M tile, batched, or head-major output): persistent,
// warp-specialized, ping-pong.  grid = min(tiles, SMs), 384 threads:
//   warpgroup 0      producer: one TMA lane (setmaxnreg lowered); walks the CTA's tiles t = blockIdx.x + i * gridDim.x
//                    in M-grouped raster order and keeps the ring full ACROSS tile boundaries
//   warpgroups 1, 2  consumers (setmaxnreg raised): consumer c owns the CTA's tiles i = c, c + 2, ...: a whole 128 x 128
//                    tile, 2 x wgmma.m64n128k16 x 3 terms per k16 step into 128 accumulator registers per thread.  An
//                    ordered pair of named barriers makes the two main loops alternate, so one consumer's register-
//                    direct epilogue runs while the other one's main loop holds the tensor cores.
//
// gemm_tc_split_kernel<WG> (decode time: one M tile, unbatched).  One CTA per 128-column tile: WG consumer warpgroups
// read an A box of 64 * WG rows, warpgroup wg consumes rows 64*wg .. 64*wg+63 (one m64n128k16 x 3 terms per k16 step),
// and warp 4 * WG is the TMA lane.  WG = 1 serves M <= 64 (a decode step of a session of at most 64 windows: no wgmma
// on zero-filled rows) with a 4-stage ring of 48 KB stages, WG = 2 serves 65..128 rows with 3 stages of 64 KB.  These
// GEMMs are weight-bandwidth bound, and with one CTA per 128-column tile too few SMs would stream the weights.  So K is
// split over the CTAs of a thread-block CLUSTER (grid z = S, cluster = (1, 1, S), S <= 8): each CTA parks its float32
// partial tile in its own shared memory (the idle operand ring), the cluster synchronises, and CTA r reduces rows
// r, r + S, ... of all S partials over distributed shared memory (4 columns per 16-byte ld.shared::cluster) and applies
// the epilogue to them: no atomics, no global workspace, a fixed summation order (bit-reproducible), and the epilogue
// itself is spread over S SMs.  A CTA streams only 2..10 k-blocks (20 for the vocabulary projection), so its time is
// round trips to HBM, not bytes: with WtsGemm::b_const the producer issues the weight (B) boxes of the first ring stages
// before the dependency wait, so the whole share of a D x D GEMM's CTA and most of a QKV / FC1 CTA's are in flight while
// the previous kernel runs.  Nothing of a row's arithmetic depends on WG: both instances give the same bits.
#include <cuda_bf16.h>

#include "sm90.cuh"

namespace wts {

constexpr int BM = 128, BN = 128, BK = 64;
constexpr int TILE_BYTES = BM * BK * 2;                 // 16 KB: one 128 x 64 bf16 box
constexpr int STAGES = 3;
constexpr int STAGE_BYTES = 4 * TILE_BYTES;
constexpr int PT_THREADS = 384;                         // persistent kernel: producer + 2 consumer warpgroups
constexpr int PT_PRODUCER_REGS = 40, PT_CONSUMER_REGS = 232;
static_assert(128 * PT_PRODUCER_REGS + 256 * PT_CONSUMER_REGS <= 65536, "setmaxnreg plan exceeds the register file");
constexpr int GROUP_M = 8;                              // M tiles per raster group of the persistent scheduler
constexpr int GT_SMEM = STAGES * STAGE_BYTES + 256 + 1024;
constexpr int PART_LD = BN + 4;                         // float pitch of a parked partial tile

// what differs between the two instances of gemm_tc_split_kernel
template <int WG>
struct SplitTraits {
    static constexpr int A_BYTES = 64 * WG * BK * 2;
    static constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * TILE_BYTES;   // A_hi, A_lo, B_hi, B_lo
    static constexpr int STAGES = WG == 1 ? 4 : 3;      // measured for WG = 1: 2 and 3 stages are slower
    static constexpr int THREADS = 128 * WG + 32;       // the consumer warpgroups + the TMA warp
    static_assert(STAGES * STAGE_BYTES + 256 + 1024 == GT_SMEM, "a 192 KB ring: the persistent kernel's shared memory");
    static_assert(64 * WG * PART_LD * 4 <= STAGES * STAGE_BYTES, "the partial tile lives in the operand ring");
};

__device__ __forceinline__ float gelu_erf_tc(float v) { return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f)); }

struct TcArgs {
    WtsGemm g;
    int a_has_bo, a_has_bi, b_has_bo, b_has_bi;   // 0 => that batch stride is 0 (operand shared): coordinate 0
    int split_k;                                  // CTAs of a cluster that share one output tile (1 = no split)
    int pair_stores;                              // no row mask; every even column pair is one aligned store in one head
};

__device__ __forceinline__ int64_t out_offset(const WtsGemm& g, int m, int n, int64_t ld)
{
    return g.head_dim > 0 ? (int64_t)(n / g.head_dim) * g.head_stride + (int64_t)m * ld + (n % g.head_dim)
                          : (int64_t)m * ld + n;
}

__device__ __forceinline__ void store_one(const WtsGemm& g, int m, int n, float t, float* of, __nv_bfloat16* ob)
{
    if (of) of[out_offset(g, m, n, g.ldc)] = t;
    if (ob) {
        const __nv_bfloat16 hi = __float2bfloat16_rn(t);
        __nv_bfloat16* d = ob + out_offset(g, m, n, g.ldo);
        d[0] = hi;
        d[g.o_plane] = __float2bfloat16_rn(t - __bfloat162float(hi));
    }
}

// alpha/bias/GELU/residual of output columns n, n+1 (n even; n + 1 only if two) of one row
__device__ __forceinline__ float2 pair_values(const WtsGemm& g, int n, bool two, float v0, float v1, float bias_m, const float* res)
{
    float t0 = g.alpha * v0, t1 = g.alpha * v1;
    if (g.bias) {
        t0 += g.bias_on_m ? bias_m : g.bias[n];
        if (two) t1 += g.bias_on_m ? bias_m : g.bias[n + 1];
    }
    if (g.act == 1) { t0 = gelu_erf_tc(t0); t1 = gelu_erf_tc(t1); }
    if (res) { t0 += res[n]; if (two) t1 += res[n + 1]; }
    return make_float2(t0, t1);
}

// SB16 store of an aligned pair
__device__ __forceinline__ void store_pair_sb16(__nv_bfloat16* dh, int64_t plane, float t0, float t1)
{
    const __nv_bfloat162 hi = __floats2bfloat162_rn(t0, t1);
    const __nv_bfloat162 lo = __floats2bfloat162_rn(t0 - __low2float(hi), t1 - __high2float(hi));
    *reinterpret_cast<__nv_bfloat162*>(dh) = hi;
    *reinterpret_cast<__nv_bfloat162*>(dh + plane) = lo;
}

// alpha/bias/GELU/residual + float32 and/or SB16 stores of output columns n, n+1 (n even) of row m
__device__ __forceinline__ void epilogue_pair(const WtsGemm& g, int m, int n, float v0, float v1, float bias_m,
                                              const float* res, float* of, __nv_bfloat16* ob)
{
    const bool two = n + 1 < g.N;
    const float2 t = pair_values(g, n, two, v0, v1, bias_m, res);
    const float t0 = t.x, t1 = t.y;
    const bool same_head = g.head_dim == 0 || (n % g.head_dim) + 1 < g.head_dim;
    if (!(two && same_head)) {
        store_one(g, m, n, t0, of, ob);
        if (two) store_one(g, m, n + 1, t1, of, ob);
        return;
    }
    if (of) {
        float* d = of + out_offset(g, m, n, g.ldc);
        if ((reinterpret_cast<uintptr_t>(d) & 7) == 0) *reinterpret_cast<float2*>(d) = make_float2(t0, t1);
        else { d[0] = t0; d[1] = t1; }
    }
    if (ob) {
        __nv_bfloat16* dh = ob + out_offset(g, m, n, g.ldo);
        __nv_bfloat16* dl = dh + g.o_plane;
        if (((reinterpret_cast<uintptr_t>(dh) | reinterpret_cast<uintptr_t>(dl)) & 3) == 0) {
            store_pair_sb16(dh, g.o_plane, t0, t1);
        } else {
            const __nv_bfloat162 hi = __floats2bfloat162_rn(t0, t1);
            const __nv_bfloat162 lo = __floats2bfloat162_rn(t0 - __low2float(hi), t1 - __high2float(hi));
            dh[0] = hi.x; dh[1] = hi.y; dl[0] = lo.x; dl[1] = lo.y;
        }
    }
}

// epilogue of one m64n128 accumulator fragment (rows m_base + t/4 and m_base + t/4 + 8 of lane t, see wgmma_ss_n128)
// straight from registers, output tile column origin n0, batch coordinates (zo, zi).  PAIRS: every column pair of the
// tile is inside N, inside one head and stored aligned (TcArgs::pair_stores and a whole tile): the pair code without
// the per-element fallbacks, a fraction of the instructions the epilogue has to stream through the instruction cache.
template <bool PAIRS>
__device__ __forceinline__ void epilogue_frag64(const WtsGemm& g, int zo, int zi, int m_base, int n0, const float (&acc)[64])
{
    const int lane = threadIdx.x & 31;
    const int cl = 2 * (lane & 3);                    // tile column of acc[4j]: cl + 8j
    float* of = g.out_f32 ? g.out_f32 + (int64_t)zo * g.c_bo + (int64_t)zi * g.c_bi : nullptr;
    __nv_bfloat16* ob = g.out_sb16 ? reinterpret_cast<__nv_bfloat16*>(g.out_sb16) + (int64_t)zo * g.o_bo + (int64_t)zi * g.o_bi : nullptr;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int m = m_base + (lane >> 2) + 8 * i;
        if (m >= g.M || (g.row_mask && g.row_mask[m] == 0)) continue;
        const float* res = g.residual ? g.residual + (int64_t)zo * g.r_bo + (int64_t)zi * g.r_bi + (int64_t)m * g.ldr : nullptr;
        const float bias_m = (g.bias && g.bias_on_m) ? g.bias[m] : 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int n = n0 + cl + 8 * j;
            if (PAIRS) {
                const float2 t = pair_values(g, n, true, acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1], bias_m, res);
                if (of) *reinterpret_cast<float2*>(of + out_offset(g, m, n, g.ldc)) = t;
                if (ob) store_pair_sb16(ob + out_offset(g, m, n, g.ldo), g.o_plane, t.x, t.y);
            } else if (n < g.N) {
                epilogue_pair(g, m, n, acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1], bias_m, res, of, ob);
            }
        }
    }
}

// element (m, n) of a K-split tile: the S <= 8 partials x[0..S) summed in rank order (the zeros past S add nothing),
// then the epilogue
__device__ __forceinline__ void split_epilogue_one(const WtsGemm& g, int m, int n, const float (&x)[8], float bias_n)
{
    float t = 0.f;
#pragma unroll
    for (int s = 0; s < 8; ++s) t += x[s];
    t = g.alpha * t + (g.bias ? (g.bias_on_m ? g.bias[m] : bias_n) : 0.f);
    if (g.act == 1) t = gelu_erf_tc(t);
    if (g.residual) t += g.residual[(int64_t)m * g.ldr + n];
    store_one(g, m, n, t, g.out_f32, reinterpret_cast<__nv_bfloat16*>(g.out_sb16));
}

__device__ __forceinline__ void named_bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }

struct TileCoord { int m0, n0, zo, zi; };

// tile t of the persistent schedule: batch-major; inside a batch item, groups of GROUP_M M tiles, M fastest inside a
// group, so the tiles in flight at one time share a few A row blocks and B column blocks in L2
__device__ __forceinline__ TileCoord tile_coord(const WtsGemm& g, int t, int tiles_m, int tiles_n)
{
    const int per_batch = tiles_m * tiles_n;
    const int z = t / per_batch;
    int r = t - z * per_batch;
    const int span = GROUP_M * tiles_n;
    const int grp = r / span;
    const int m_first = grp * GROUP_M;
    const int gm = min(GROUP_M, tiles_m - m_first);
    r -= grp * span;
    TileCoord c;
    c.m0 = (m_first + r % gm) * BM;
    c.n0 = (r / gm) * BN;
    c.zo = z / g.batch_inner;
    c.zi = z - c.zo * g.batch_inner;
    return c;
}

__global__ void __launch_bounds__(PT_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TcArgs args)
{
    extern __shared__ unsigned char smem_raw[];
    const WtsGemm& g = args.g;
    const uint32_t base = (smem_addr(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar = base + STAGES * STAGE_BYTES;   // full[s] at +8s, empty[s] at +32+8s
    const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int tiles_n = (g.N + BN - 1) / BN, tiles_m = (g.M + BM - 1) / BM;
    const int tiles = tiles_m * tiles_n * g.batch_outer * g.batch_inner;
    const int nkb = (g.K + BK - 1) / BK;
    pdl_launch();

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
        for (int s = 0; s < STAGES; ++s) { mbar_init(bar + 8 * s, 1); mbar_init(bar + 32 + 8 * s, 4); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pdl_wait();                                     // everything above overlapped the previous kernel's tail

    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PT_PRODUCER_REGS));
        if (warp == 0 && lane == 0) {
            int p = 0;                              // ring position: k-block p of the CTA's whole tile sequence
            for (int t = blockIdx.x; t < tiles; t += gridDim.x) {
                const TileCoord tc = tile_coord(g, t, tiles_m, tiles_n);
                const int azo = args.a_has_bo ? tc.zo : 0, azi = args.a_has_bi ? tc.zi : 0;
                const int bzo = args.b_has_bo ? tc.zo : 0, bzi = args.b_has_bi ? tc.zi : 0;
                for (int kb = 0; kb < nkb; ++kb, ++p) {
                    const int s = p % STAGES, u = p / STAGES;
                    mbar_wait(bar + 32 + 8 * s, (u & 1) ^ 1);
                    const uint32_t full = bar + 8 * s;
                    mbar_expect_tx(full, STAGE_BYTES);
                    const uint32_t st = base + s * STAGE_BYTES;
                    const int kc = kb * BK;
                    tma_load_5d(st, &tmA, full, kc, tc.m0, azi, azo, 0);
                    tma_load_5d(st + TILE_BYTES, &tmA, full, kc, tc.m0, azi, azo, 1);
                    tma_load_5d(st + 2 * TILE_BYTES, &tmB, full, kc, tc.n0, bzi, bzo, 0);
                    tma_load_5d(st + 3 * TILE_BYTES, &tmB, full, kc, tc.n0, bzi, bzo, 1);
                }
            }
        }
        return;
    }

    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(PT_CONSUMER_REGS));
    const int c = wg - 1;                           // consumer 0 / 1: the CTA's even / odd tiles
    float acc[2][64];
    int l = c;                                      // index of the tile in the CTA's sequence
    for (int t = blockIdx.x + c * gridDim.x; t < tiles; t += 2 * gridDim.x, l += 2) {
        // named barrier 1 + c: "consumer c may start its main loop", arrived by the other consumer
        if (l > 0) named_bar_sync(1 + c, 256);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 64; ++i) acc[h][i] = 0.f;
        int p = l * nkb;
        for (int kb = 0; kb < nkb; ++kb, ++p) {
            const int s = p % STAGES;
            mbar_wait(bar + 8 * s, (p / STAGES) & 1);
            const uint32_t st = base + s * STAGE_BYTES;
            const uint64_t a_hi = wg_desc(st), a_lo = wg_desc(st + TILE_BYTES);
            const uint64_t b_hi = wg_desc(st + 2 * TILE_BYTES), b_lo = wg_desc(st + 3 * TILE_BYTES);
            constexpr uint64_t a_half = (TILE_BYTES / 2) >> 4;   // rows 64..127 of an A box, in 16-byte units
            wg_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                const uint64_t adv = (uint64_t)(k * 2);       // 32 bytes per K=16 step, in 16-byte units
#pragma unroll
                for (int h = 0; h < 2; ++h) wgmma_ss_n128(acc[h], a_hi + h * a_half + adv, b_hi + adv, 1);
#pragma unroll
                for (int h = 0; h < 2; ++h) wgmma_ss_n128(acc[h], a_lo + h * a_half + adv, b_hi + adv, 1);
#pragma unroll
                for (int h = 0; h < 2; ++h) wgmma_ss_n128(acc[h], a_hi + h * a_half + adv, b_lo + adv, 1);
            }
            wg_commit();
            wg_wait<1>();                                     // the previous k-block's wgmmas have retired
            if (kb > 0 && lane == 0) mbar_arrive(bar + 32 + 8 * ((p - 1) % STAGES));
        }
        // every wgmma of this tile is issued: the other consumer's main loop may start (if it has a next tile)
        if (t + gridDim.x < tiles) named_bar_arrive(2 - c, 256);
        wg_wait<0>();
        if (lane == 0) mbar_arrive(bar + 32 + 8 * ((p - 1) % STAGES));

        const TileCoord tc = tile_coord(g, t, tiles_m, tiles_n);
        const bool pairs = args.pair_stores && tc.n0 + BN <= g.N;
        // not unrolled over the two halves: one copy of the epilogue code, fed by a register select
#pragma unroll 1
        for (int h = 0; h < 2; ++h) {
            float v[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) v[i] = h ? acc[1][i] : acc[0][i];
            if (pairs) epilogue_frag64<true>(g, tc.zo, tc.zi, tc.m0 + 64 * h + 16 * warp, tc.n0, v);
            else epilogue_frag64<false>(g, tc.zo, tc.zi, tc.m0 + 64 * h + 16 * warp, tc.n0, v);
        }
    }
}

template <int WG>
__global__ void __launch_bounds__(SplitTraits<WG>::THREADS, 1)
gemm_tc_split_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TcArgs args)
{
    using T = SplitTraits<WG>;
    extern __shared__ unsigned char smem_raw[];
    const WtsGemm& g = args.g;
    const uint32_t base = (smem_addr(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar = base + T::STAGES * T::STAGE_BYTES;   // full[s] at +8s, empty[s] at +32+8s
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n0 = blockIdx.x * BN;
    const int S = args.split_k;
    const int nkb_all = (g.K + BK - 1) / BK;
    const int kb0 = (int)((int64_t)blockIdx.z * nkb_all / S);
    const int nkb = (int)((int64_t)(blockIdx.z + 1) * nkb_all / S) - kb0;
    pdl_launch();

    if (threadIdx.x == 128 * WG) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
        for (int s = 0; s < T::STAGES; ++s) { mbar_init(bar + 8 * s, 1); mbar_init(bar + 32 + 8 * s, 4 * WG); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    float acc[64];
    if (warp == 4 * WG) {
        if (lane == 0) {
            // the weights are not written by any earlier kernel of the stream: the first stages' B boxes are issued
            // before the dependency wait, their A (activation) boxes after it, on the same full barriers
            const int pre = g.b_const ? min(nkb, T::STAGES) : 0;
            for (int kb = 0; kb < pre; ++kb) {
                const uint32_t st = base + kb * T::STAGE_BYTES, full = bar + 8 * kb;
                mbar_expect_tx(full, T::STAGE_BYTES);
                tma_load_5d(st + 2 * T::A_BYTES, &tmB, full, (kb0 + kb) * BK, n0, 0, 0, 0);
                tma_load_5d(st + 2 * T::A_BYTES + TILE_BYTES, &tmB, full, (kb0 + kb) * BK, n0, 0, 0, 1);
            }
            pdl_wait();
            for (int kb = 0; kb < pre; ++kb) {
                const uint32_t st = base + kb * T::STAGE_BYTES, full = bar + 8 * kb;
                tma_load_5d(st, &tmA, full, (kb0 + kb) * BK, 0, 0, 0, 0);
                tma_load_5d(st + T::A_BYTES, &tmA, full, (kb0 + kb) * BK, 0, 0, 0, 1);
            }
            for (int kb = pre; kb < nkb; ++kb) {
                const int s = kb % T::STAGES, u = kb / T::STAGES;
                mbar_wait(bar + 32 + 8 * s, (u & 1) ^ 1);
                const uint32_t full = bar + 8 * s;
                mbar_expect_tx(full, T::STAGE_BYTES);
                const uint32_t st = base + s * T::STAGE_BYTES;
                const int kc = (kb0 + kb) * BK;
                tma_load_5d(st, &tmA, full, kc, 0, 0, 0, 0);
                tma_load_5d(st + T::A_BYTES, &tmA, full, kc, 0, 0, 0, 1);
                tma_load_5d(st + 2 * T::A_BYTES, &tmB, full, kc, n0, 0, 0, 0);
                tma_load_5d(st + 2 * T::A_BYTES + TILE_BYTES, &tmB, full, kc, n0, 0, 0, 1);
            }
        } else {
            pdl_wait();
        }
    } else {
        pdl_wait();                                 // the epilogue reads bias / residual / row mask written upstream
        // the warpgroup's 64 rows of an A box; a literal 0 for WG = 1, where the compiler cannot infer warp < 4
        const uint32_t a_rows = (WG == 1 ? 0 : warp >> 2) * (T::A_BYTES / WG);
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        for (int kb = 0; kb < nkb; ++kb) {
            const int s = kb % T::STAGES, u = kb / T::STAGES;
            mbar_wait(bar + 8 * s, u & 1);
            const uint32_t st = base + s * T::STAGE_BYTES;
            const uint64_t a_hi = wg_desc(st + a_rows), a_lo = wg_desc(st + T::A_BYTES + a_rows);
            const uint64_t b_hi = wg_desc(st + 2 * T::A_BYTES), b_lo = wg_desc(st + 2 * T::A_BYTES + TILE_BYTES);
            wg_fence();
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) {
                const uint64_t adv = (uint64_t)(k * 2);       // 32 bytes per K=16 step, in 16-byte units
                wgmma_ss_n128(acc, a_hi + adv, b_hi + adv, 1);
                wgmma_ss_n128(acc, a_lo + adv, b_hi + adv, 1);
                wgmma_ss_n128(acc, a_hi + adv, b_lo + adv, 1);
            }
            wg_commit();
            wg_wait<1>();                                     // the previous k-block's wgmmas have retired
            if (kb > 0 && lane == 0) mbar_arrive(bar + 32 + 8 * ((kb - 1) % T::STAGES));
        }
        wg_wait<0>();

        if (S == 1) {
            epilogue_frag64<false>(g, 0, 0, 16 * warp, n0, acc);
        } else {
            // the ring is idle once every consumer warpgroup has retired its wgmmas (every TMA write has landed: all
            // full barriers were waited)
            asm volatile("bar.sync 1, %0;" ::"n"(128 * WG) : "memory");
            float* part = reinterpret_cast<float*>(smem_raw + (base - smem_addr(smem_raw)));
            const int rl = 16 * warp + (lane >> 2), cl = 2 * (lane & 3);
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 16; ++j)
                    *reinterpret_cast<float2*>(part + (rl + 8 * i) * PART_LD + cl + 8 * j) =
                        make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
        }
    }
    if (S > 1) {
        __syncwarp();
        cluster_sync_all();                          // every partial tile is parked and visible cluster-wide
        if (threadIdx.x < 128 * WG) {
            // CTA r reduces rows r + S * (4 * WG * i + warp); a lane owns 4 adjacent columns and reads them from each
            // of the S partial tiles with one 16-byte distributed-shared-memory load
            uint32_t rank;
            asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
            const int c = 4 * lane, n = n0 + c;
            if (n < g.N) {
                uint32_t peer[8];
#pragma unroll
                for (int s = 0; s < 8; ++s) {
                    peer[s] = 0;
                    if (s < S) asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer[s]) : "r"(base + 4u * c), "r"(s));
                }
                float bias_n[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) bias_n[e] = (g.bias && !g.bias_on_m && n + e < g.N) ? g.bias[n + e] : 0.f;
#pragma unroll 1
                for (int m = (int)rank + S * warp; m < g.M; m += 4 * WG * S) {
                    if (g.row_mask && g.row_mask[m] == 0) continue;
                    float x[4][8];
#pragma unroll
                    for (int s = 0; s < 8; ++s) {
                        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (s < S)
                            asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];"
                                         : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                                         : "r"(peer[s] + (uint32_t)(m * PART_LD * 4)));
                        x[0][s] = v.x; x[1][s] = v.y; x[2][s] = v.z; x[3][s] = v.w;
                    }
#pragma unroll
                    for (int e = 0; e < 4; ++e)
                        if (n + e < g.N) split_epilogue_one(g, m, n + e, x[e], bias_n[e]);
                }
            }
        }
        __syncwarp();
        cluster_sync_all();                          // nobody leaves while a peer may still read its partial tile
    }
}

// ---------------------------------------------------------------------------------------- host side
// 5-D bf16 map: (K, rows, inner batch, outer batch, plane); strides in ELEMENTS
static int make_map(CUtensorMap* tm, const void* ptr, int64_t K, int64_t rows, int64_t ld, int64_t plane, int64_t n_bi,
                    int64_t s_bi, int64_t n_bo, int64_t s_bo, int box_rows, const char* which)
{
    auto enc = tensor_map_encoder();
    if (!enc) { set_error("wts_gemm: cuTensorMapEncodeTiled entry point not available"); return -4; }
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (ld & 7) || (plane & 7) || (s_bi & 7) || (s_bo & 7)) {
        set_error("wts_gemm(tc): operand %s not 16-byte aligned (ptr=%p ld=%lld plane=%lld bi=%lld bo=%lld)", which, ptr,
                  (long long)ld, (long long)plane, (long long)s_bi, (long long)s_bo);
        return -5;
    }
    const int64_t e_bi = s_bi ? n_bi : 1, e_bo = s_bo ? n_bo : 1;
    cuuint64_t dims[5] = {(cuuint64_t)K, (cuuint64_t)rows, (cuuint64_t)e_bi, (cuuint64_t)e_bo, 2};
    const cuuint64_t row_b = (cuuint64_t)ld * 2;
    cuuint64_t strides[4] = {row_b, (cuuint64_t)(s_bi ? s_bi * 2 : row_b), (cuuint64_t)(s_bo ? s_bo * 2 : row_b),
                             (cuuint64_t)plane * 2};
    cuuint32_t box[5] = {BK, (cuuint32_t)box_rows, 1, 1, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("wts_gemm(tc): cuTensorMapEncodeTiled(%s) failed with %d (K=%lld rows=%lld ld=%lld plane=%lld)", which, (int)r,
                  (long long)K, (long long)rows, (long long)ld, (long long)plane);
        return -6;
    }
    return 0;
}

int gemm_tc_launch(const WtsGemm& g, cudaStream_t st)
{
    static int n_sm = 0;
    if (n_sm == 0) {
        for (auto kernel : {gemm_tc_kernel, gemm_tc_split_kernel<1>, gemm_tc_split_kernel<2>})
            WTS_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GT_SMEM));
        int dev = 0;
        WTS_CUDA_CHECK(cudaGetDevice(&dev));
        WTS_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    }
    const int tiles_n = (g.N + BN - 1) / BN, tiles_m = (g.M + BM - 1) / BM, nkb = (g.K + BK - 1) / BK;
    const int batch = g.batch_outer * g.batch_inner;
    const bool skinny = tiles_m == 1 && batch == 1 && g.head_dim == 0;
    const int wg = g.M <= 64 ? 1 : 2;                 // consumer warpgroups of the split kernel
    alignas(64) CUtensorMap tmA, tmB;
    int rc = make_map(&tmA, g.a, g.K, g.M, g.lda, g.a_plane, g.batch_inner, g.a_bi, g.batch_outer, g.a_bo,
                      skinny ? 64 * wg : BM, "A");
    if (rc) return rc;
    rc = make_map(&tmB, g.b, g.K, g.N, g.ldb, g.b_plane, g.batch_inner, g.b_bi, g.batch_outer, g.b_bo, BN, "B");
    if (rc) return rc;
    TcArgs args;
    args.g = g;
    args.a_has_bo = g.a_bo != 0; args.a_has_bi = g.a_bi != 0;
    args.b_has_bo = g.b_bo != 0; args.b_has_bi = g.b_bi != 0;
    cudaLaunchConfig_t cfg = {};
    cfg.dynamicSmemBytes = GT_SMEM;
    cfg.stream = st;
    if (!skinny) {
        const int64_t tiles = (int64_t)tiles_m * tiles_n * batch;
        if (tiles > INT32_MAX / 2) { set_error("wts_gemm(tc): %lld output tiles are too many", (long long)tiles); return -7; }
        args.split_k = 1;
        const bool heads_even = g.head_dim == 0 || (g.head_dim % 2 == 0 && g.head_stride % 2 == 0);
        const bool of_pairs = !g.out_f32 || ((reinterpret_cast<uintptr_t>(g.out_f32) & 7) == 0 && g.ldc % 2 == 0 &&
                                             g.c_bo % 2 == 0 && g.c_bi % 2 == 0);
        const bool ob_pairs = !g.out_sb16 || ((reinterpret_cast<uintptr_t>(g.out_sb16) & 3) == 0 && g.ldo % 2 == 0 &&
                                              g.o_plane % 2 == 0 && g.o_bo % 2 == 0 && g.o_bi % 2 == 0);
        args.pair_stores = !g.row_mask && heads_even && of_pairs && ob_pairs;
        cfg.gridDim = dim3((unsigned)(tiles < n_sm ? tiles : n_sm), 1, 1);
        cfg.blockDim = dim3(PT_THREADS, 1, 1);
        WTS_CUDA_CHECK(cudaLaunchKernelEx(&cfg, gemm_tc_kernel, tmA, tmB, args));
        return 0;
    }
    int split = 1;
    if (2 * tiles_n <= n_sm) {
        split = n_sm / tiles_n;
        if (split > 8) split = 8;                     // portable cluster size
        if (split > nkb) split = nkb;
    }
    args.split_k = split;
    args.pair_stores = 0;
    cfg.gridDim = dim3(tiles_n, 1, split);
    cfg.blockDim = dim3(wg == 1 ? SplitTraits<1>::THREADS : SplitTraits<2>::THREADS, 1, 1);
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (split > 1) {
        attr[na].id = cudaLaunchAttributeClusterDimension;
        attr[na].val.clusterDim.x = 1;
        attr[na].val.clusterDim.y = 1;
        attr[na].val.clusterDim.z = split;
        ++na;
    }
    if (pdl_enabled()) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    WTS_CUDA_CHECK(cudaLaunchKernelEx(&cfg, wg == 1 ? gemm_tc_split_kernel<1> : gemm_tc_split_kernel<2>, tmA, tmB, args));
    return 0;
}

}  // namespace wts
