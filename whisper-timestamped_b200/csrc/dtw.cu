// Batched monotonic DTW (symmetric1) as a warp-wavefront kernel for sm_90a.
//
// Replaces  dtw.dtw(weights, step_pattern=dtw.stepPattern.symmetric1)   (T.py:1572-1581)
// and the jumps extraction                                              (T.py:1648-1652)
// where T.py = /root/reference/whisper_timestamped/transcribe.py.
//
// Semantics restated from dtw-python (see oracle/dtw_oracle.c): for every cell the three
// candidates  cm[i-1,j-1]+lm, cm[i,j-1]+lm, cm[i-1,j]+lm  are formed in float64 (one add each) and
// the FIRST strict minimum wins (diag < left < up on ties).  Every cell depends only on its
// three predecessors, so an anti-diagonal wavefront produces bit-identical cm / directions.
//
// Mapping: one warp per cost matrix.  Lane L (1..31) owns matrix row row0+L-1 of the current
// 31-row strip and walks it left to right; at step s it sits on column j = s-(L-1), i.e. the
// warp sweeps anti-diagonals.  Lane 0 plays the row above the strip (+inf for the first strip,
// the previous strip's last row otherwise), so `up` is one shfl_up and `diag` is last step's
// `up`; +inf stands for dtw-python's NaN "no predecessor" (never wins a strict '<').
// Local costs are staged through shared memory: each 32-column tile is fetched from HBM with
// fully coalesced 128-byte row segments by cp.async (LDGSTS) 31 steps before it is consumed and
// parked in a 64-slot circular row buffer, SKEWED by the row index: element (row L, column j)
// lives in slot (j+L-1)&63 = s&63, so the read of step s is `row_base + 4*(s&63)` for every lane
// (an immediate offset, no address arithmetic in the dependent chain) and the odd row pitch of 65
// words puts the 32 lanes on 32 distinct banks.  Directions are packed 2 bits/cell in "skewed" words (field = step index),
// one coalesced 128-byte store per 16 steps.  The backtrack then needs one step per TOKEN ROW
// (not per path cell): find the previous non-horizontal move with a clz on the packed words.
#include "common.cuh"

namespace wts {

constexpr int RS = 31;         // matrix rows per strip (lanes 1..31)
constexpr int DTW_WARPS = 2;   // warps (= matrices) per CTA
constexpr int DS_WORDS = 24;   // direction words per lane row kept in shared memory (covers F <= 354 single-strip)
constexpr int RING = 64;       // slots per lane row: 2 tiles of 32 columns
constexpr int PITCH = RING + 1; // odd row pitch (words): the 32 lanes of a diagonal read hit 32 banks
constexpr int TILE_WORDS = 33 * 64;           // per-warp staging buffer (32 rows x 65 <= 33*64), 256-B multiple
#ifndef DTW_MIN_CTAS
#define DTW_MIN_CTAS 9
#endif

__host__ __device__ inline int dtw_nstrips(int T) { return (T + RS - 1) / RS; }
__host__ __device__ inline int dtw_niter(int F) { return (F + RS - 1 + 31) / 32; }
__host__ __device__ inline int dtw_wpr(int F) { return 2 * dtw_niter(F); }   // dir words per lane row

// segments the single-strip fast path (dtw_small_kernel, below) takes over from the general kernel
__host__ __device__ inline bool dtw_small_eligible(const WtsSegDesc& sd)
{
    return (sd.flags & (WTS_SEG_NONPOSITIVE | WTS_SEG_PITCH16)) == (WTS_SEG_NONPOSITIVE | WTS_SEG_PITCH16) &&
           sd.T >= 1 && sd.T <= RS && sd.F >= 1 && dtw_wpr(sd.F) <= DS_WORDS;
}

// segments the lane-per-matrix path (dtw_lane_kernel<TR>, below) owns when a call uses it
__host__ __device__ inline bool dtw_lane_eligible(const WtsSegDesc& sd, int TR)
{
    return (sd.flags & (WTS_SEG_NONPOSITIVE | WTS_SEG_PITCH16)) == (WTS_SEG_NONPOSITIVE | WTS_SEG_PITCH16) &&
           sd.T >= 1 && sd.T <= TR && sd.F >= 1;
}

__device__ __forceinline__ double dinf() { return __longlong_as_double(0x7ff0000000000000LL); }

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
template <typename TIn> __device__ __forceinline__ TIn lds(uint32_t addr);
template <> __device__ __forceinline__ float lds<float>(uint32_t addr) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory"); return v; }
template <> __device__ __forceinline__ double lds<double>(uint32_t addr) { double v; asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(addr) : "memory"); return v; }
template <int BYTES> __device__ __forceinline__ void cp_async(uint32_t dst, const void* src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(dst), "l"(src), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// One 31-row strip.  Staging: row k of the next 32-column tile is fetched with one warp-wide cp.async (LDGSTS)
// at step k of the current tile, i.e. 31 steps before its first use, into a 64-slot ring per row, skewed by the
// row index: element (row L, column j) lives in slot (j+L-1)&63 = step&63, so step s reads
// `row_base + (s&63)*ES` for every lane (immediate offsets; the odd row pitch gives 32 distinct banks).  The slot a
// row overwrites was last read two steps earlier.  Two commit groups per tile (rows 1-15, rows 16-31) keep every
// wait_group at least 16 steps behind its loads.  Loads are clamped (column to F-1, rows beyond the strip skipped)
// so every issued address is valid; cells outside the matrix only see finite values and are never consumed.
//
// NEG: all local costs are <= 0 and cost[0,0] < 0 (what the attention post-processing produces), hence every
// accumulated cost is a strictly negative double (or +inf for "no predecessor") and  a < b  <=>  bits(a) >u bits(b).
// The two fp64 compares of the dependent chain become integer compares (same results bit for bit).
template <typename TIn, bool FIRST, bool WRITE_BND, bool NEG>
__device__ __forceinline__ void dtw_fill_strip(const TIn* __restrict__ C, const int F, const int P, const int row0,
                                               const int Ts, const int niter, const uint32_t tile_a,
                                               uint32_t* __restrict__ dirs_strip,
                                               double* __restrict__ bnd, const int lane)
{
    constexpr uint32_t ES = sizeof(TIn);
    constexpr uint32_t ROWB = PITCH * ES;
    constexpr uint32_t SLOTMASK = (RING - 1) * ES;
    const double INF = dinf();
    double cur = INF, upprev = INF;
    if (FIRST && lane == 1) upprev = 0.0;            // seeds cm[0,0] = 0 + lm[0,0]
    if (!FIRST && lane == 0) cur = __ldcg(bnd);      // cm[row0-1, 0]
    uint32_t acc = 0;
    const uint32_t myrow_a = tile_a + lane * ROWB;
    const uint32_t laneb = lane * ES;
    const char* Cb = reinterpret_cast<const char*>(C + (int64_t)row0 * P);   // strip row 0 (= tile row 1); P = row pitch
    const uint32_t Fb = (uint32_t)P * ES;

    // prologue: tile 0 (all rows), one group
    {
        const char* src = Cb + (uint32_t)min(lane, F - 1) * ES;
        for (int k = 1; k <= Ts; ++k) {
            cp_async<ES>(tile_a + k * ROWB + ((laneb + (uint32_t)(k - 1) * ES) & SLOTMASK), src);
            src += Fb;
        }
        cp_async_commit();
    }
    double bndreg = INF, bndnext = INF;
    if (!FIRST) {
        const int idx = 1 + lane;
        bndnext = idx < F ? __ldcg(bnd + idx) : INF;
    }

    for (int t = 0; t < niter; ++t) {
        if (!FIRST) {
            bndreg = bndnext;
            const int idx = 32 * (t + 1) + 1 + lane;
            bndnext = idx < F ? __ldcg(bnd + idx) : INF;
        }
        // tile t: rows 1..15 were committed >= 16 steps ago (group A), rows 16..31 are group B (waited at k = 15)
        if (t == 0) cp_async_wait<0>(); else cp_async_wait<1>();
        __syncwarp();
        const uint32_t rd_a = myrow_a + (uint32_t)((32 * t) & (RING - 1)) * ES;
        const uint32_t slot0 = laneb + (uint32_t)(32 * (t + 1) + RING - 1) * ES;   // (+RING-1 == -1 mod RING)
        const char* src = Cb + (uint32_t)min(32 * (t + 1) + lane, F - 1) * ES;
#pragma unroll
        for (int k = 0; k < 32; ++k) {
            if (k >= 1 && k <= Ts) {                  // row k of tile t+1; its slot was last read at step k-2
                cp_async<ES>(tile_a + k * ROWB + ((slot0 + k * ES) & SLOTMASK), src);
                src += Fb;
            }
            if (k == 15) { cp_async_commit(); cp_async_wait<1>(); __syncwarp(); }   // group A out; tile t group B landed
            // ---- one anti-diagonal
            const int s = 32 * t + k;
            const double l = (double)lds<TIn>(rd_a + k * ES);
            const double up = __shfl_up_sync(FULL_MASK, cur, 1);
            const double diag = upprev;
            upprev = up;
            const double c1 = diag + l, c2 = cur + l, c3 = up + l;
            bool p2, p3;
            double m, best;
            if (NEG) {
                p2 = (unsigned long long)__double_as_longlong(c2) > (unsigned long long)__double_as_longlong(c1);
                m = p2 ? c2 : c1;
                p3 = (unsigned long long)__double_as_longlong(c3) > (unsigned long long)__double_as_longlong(m);
                best = p3 ? c3 : m;
            } else {
                p2 = c2 < c1;                         // left beats diag
                m = p2 ? c2 : c1;
                p3 = c3 < m;                          // up beats both
                best = p3 ? c3 : m;
            }
            cur = best;
            if ((k & 15) == 0) acc = 0;
            if (p2) acc |= 1u << (2 * (k & 15));
            if (p3) acc |= 2u << (2 * (k & 15));
            if ((k & 15) == 15) dirs_strip[(2 * t + (k >> 4)) * 32 + lane] = acc;
            if (WRITE_BND) {
                const int j = s - (Ts - 1);
                if (lane == Ts && j >= 0 && j < F) bnd[j] = best;
            }
            if (!FIRST) {
                const double ub = __shfl_sync(FULL_MASK, bndreg, k);
                if (lane == 0) cur = ub;             // cm[row0-1, s+1]
            }
        }
        cp_async_commit();                            // group B of tile t+1
    }
    cp_async_wait<0>();
}

// Direction fields (2 bits per cell, field index = step & 15): bit0 = "left beats diag",
// bit1 = "up beats both".  up if bit1, else left if bit0, else diag.
__device__ __forceinline__ uint32_t dtw_nonleft_mask(uint32_t x)
{
    const uint32_t lo = x & 0x55555555u, hi = (x >> 1) & 0x55555555u;
    return 0x55555555u & ~(lo & ~hi);
}

// ---- backtrack, one step per token row (executed redundantly by all lanes; lane 0 stores): jumps[i] = first path
// column of token row i (T.py:1648-1652), jumps[T] = F - 1.
__device__ __forceinline__ void dtw_backtrack_jumps(const uint32_t* dirs, const int W, const int T, const int F,
                                                    int32_t* __restrict__ jumps, const int lane)
{
    int i = T - 1, j = F - 1;
    if (lane == 0) jumps[T] = F - 1;
    while (i > 0) {
        const int strip = i / RS, ln = i - strip * RS + 1;
        const uint32_t* base = dirs + (int64_t)strip * W * 32 + ln;
        int s = j + ln - 1;
        int w = s >> 4, pos = s & 15, kf = 0;
        uint32_t x = 0;
        while (true) {
            x = base[w * 32];
            const uint32_t m = dtw_nonleft_mask(x) & (0xffffffffu >> (30 - 2 * pos));
            if (m) { kf = (31 - __clz(m)) >> 1; break; }
            if (w == 0) { kf = 0; break; }
            --w; pos = 15;
        }
        int jj = w * 16 + kf - (ln - 1);
        if (jj < 0) jj = 0;
        const bool is_up = (x >> (2 * kf + 1)) & 1u;
        if (lane == 0) jumps[i] = jj;
        j = (!is_up && jj > 0) ? jj - 1 : jj;       // diag or up into the previous row
        --i;
    }
    if (lane == 0) jumps[0] = 0;
}

// dir field of cell (i, j)
__device__ __forceinline__ uint32_t dtw_dir_at(const uint32_t* dirs, int W, int i, int j)
{
    const int strip = i / RS, ln = i - strip * RS + 1;
    const int s = j + ln - 1;
    const uint32_t x = dirs[((int64_t)strip * W + (s >> 4)) * 32 + ln];
    const uint32_t f = (x >> (2 * (s & 15))) & 3u;
    return (f & 2u) ? 3u : ((f & 1u) ? 2u : 1u);
}

template <typename TIn>
__global__ void __launch_bounds__(DTW_WARPS * 32, DTW_MIN_CTAS)
dtw_warp_kernel(const TIn* __restrict__ cost, const WtsSegDesc* __restrict__ segs, const int nseg,
                uint32_t* __restrict__ dir_ws, double* __restrict__ bnd_ws,
                int32_t* __restrict__ jumps_out, int32_t* __restrict__ path_out,
                const int64_t* __restrict__ path_off, int32_t* __restrict__ path_len, const int skip_small)
{
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    TIn* tile = reinterpret_cast<TIn*>(smem_raw) + warp * TILE_WORDS;
    const uint32_t tile_a = smem_u32(tile);
    uint32_t* dirs_sm = reinterpret_cast<uint32_t*>(smem_raw + (size_t)DTW_WARPS * TILE_WORDS * sizeof(TIn)) + warp * (DS_WORDS * 32);
    const int seg = blockIdx.x * DTW_WARPS + warp;
    if (seg >= nseg) return;

    const WtsSegDesc sd = segs[seg];
    // skip_small = lane-path rows << 16 | fast-path rows << 8 | fast-path dir words: segments another kernel of this call owns
    if ((skip_small >> 16) & 255) {
        if (dtw_lane_eligible(sd, (skip_small >> 16) & 255)) return;                   // dtw_lane_kernel
    } else if (skip_small && dtw_small_eligible(sd) && sd.T + 1 <= ((skip_small >> 8) & 255) && dtw_wpr(sd.F) <= (skip_small & 255)) {
        return;                                                                         // dtw_small_kernel
    }
    const int T = sd.T, F = sd.F, P = seg_pitch(sd);
    const TIn* C = cost + sd.cost_off;
    // directions live in shared memory when the whole matrix fits one strip and DS_WORDS words per row
    // (the typical alignment problem): the row-wise backtrack then never waits on L2
    uint32_t* dirs = (sd.T <= RS && dtw_wpr(sd.F) <= DS_WORDS) ? dirs_sm : dir_ws + sd.dir_off;
    double* bnd = bnd_ws + sd.bnd_off;
    int32_t* jumps = jumps_out + sd.jumps_off;
    if (T <= 0 || F <= 0) return;

    // zero the staging buffer once: cells read before their tile arrives (j < 0) must be finite
    for (int k = lane; k < TILE_WORDS; k += 32) tile[k] = TIn(0);
    __syncwarp();

    const int niter = dtw_niter(F);
    const int W = 2 * niter;
    const int nstrips = dtw_nstrips(T);
    for (int strip = 0; strip < nstrips; ++strip) {
        const int row0 = strip * RS;
        const int Ts = min(RS, T - row0);
        uint32_t* ds = dirs + (int64_t)strip * W * 32;
        const bool more = strip + 1 < nstrips;
        const bool neg = (sizeof(TIn) == 4) && (sd.flags & 1);
        if (neg) {
            if (strip == 0) {
                if (more) dtw_fill_strip<TIn, true, true, true>(C, F, P, row0, Ts, niter, tile_a, ds, bnd, lane);
                else      dtw_fill_strip<TIn, true, false, true>(C, F, P, row0, Ts, niter, tile_a, ds, bnd, lane);
            } else {
                if (more) dtw_fill_strip<TIn, false, true, true>(C, F, P, row0, Ts, niter, tile_a, ds, bnd, lane);
                else      dtw_fill_strip<TIn, false, false, true>(C, F, P, row0, Ts, niter, tile_a, ds, bnd, lane);
            }
        } else if (strip == 0) {
            if (more) dtw_fill_strip<TIn, true, true, false>(C, F, P, row0, Ts, niter, tile_a, ds, bnd, lane);
            else      dtw_fill_strip<TIn, true, false, false>(C, F, P, row0, Ts, niter, tile_a, ds, bnd, lane);
        } else {
            if (more) dtw_fill_strip<TIn, false, true, false>(C, F, P, row0, Ts, niter, tile_a, ds, bnd, lane);
            else      dtw_fill_strip<TIn, false, false, false>(C, F, P, row0, Ts, niter, tile_a, ds, bnd, lane);
        }
        __syncwarp();
    }
    __threadfence_block();
    __syncwarp();

    dtw_backtrack_jumps(dirs, W, T, F, jumps, lane);

    // ---- optional full path (alignment.index1s / index2s), cell by cell; tests & plots only
    if (path_out != nullptr && lane == 0) {
        int32_t* p1 = path_out + path_off[seg];
        int32_t* p2 = p1 + T + F;
        int i = T - 1, j = F - 1, len = 1;
        while (i > 0 || j > 0) {
            uint32_t d = dtw_dir_at(dirs, W, i, j);
            if (i == 0) d = 2u; else if (j == 0) d = 3u;
            if (d == 1u) { --i; --j; } else if (d == 2u) { --j; } else { --i; }
            ++len;
        }
        path_len[seg] = len;
        i = T - 1; j = F - 1;
        int k = len - 1;
        p1[k] = i; p2[k] = j;
        while (i > 0 || j > 0) {
            uint32_t d = dtw_dir_at(dirs, W, i, j);
            if (i == 0) d = 2u; else if (j == 0) d = 3u;
            if (d == 1u) { --i; --j; } else if (d == 2u) { --j; } else { --i; }
            --k;
            p1[k] = i; p2[k] = j;
        }
    }
}

// ------------------------------------------------------------------------------------ single-strip fast path
// The typical alignment problem (T <= 31 tokens, F <= 354 frames, float32 costs <= 0 from wts_attn_prep_batch with rows
// padded to 16 bytes) gets its own kernel, built to spend as few issue slots per anti-diagonal as the bit-exact fp64
// recurrence allows (the general kernel above is ISSUE-bound: ~40 warp instructions per step of which the recurrence
// needs ~17):
//  * staging is 16-byte cp.async (LDGSTS.128): one warp instruction moves 8 rows x 16 columns of a tile, i.e. four
//    instructions per tile of up to 31 rows, one tile ahead, completion by cp.async groups (rows are padded to 16 bytes
//    so every chunk is aligned);
//  * the row buffers are NOT skewed: a ring of five tiles (t-2 .. t being read — the 31 lanes of skew span two
//    tiles back —, t+1 and t+2 in flight) plus a mirror of slot 0 behind the ring, so lane L reads
//    `row_base + 4 p_L + 4 k` at step k of a tile — an immediate offset with no wrap inside the tile
//    (p_L = (16 t - L + 1) mod 80 advances once per tile); row pitch 96 words: bank (p_L + k) mod 32 =
//    (1 - L + k + 16 t) mod 32 is distinct over the lanes; 15 KB of shared memory per warp (rows + directions)
//    keeps 14 warps per SM resident — the dependent fp64 chain needs them;
//  * directions stay in shared memory (2 bits per cell) for the row-wise backtrack.
// Same recurrence, same tie-breaks, same packed direction words as dtw_fill_strip<float, true, false, true>.
// Geometry of a variant <TC, LA>: TC columns per tile (= wavefront steps per iteration), LA tiles in flight ahead of the
// one being consumed.  The ring holds the tiles still being read (the current one and ceil(31 / TC) behind it: the 31
// lanes of skew), plus the LA in flight; a mirror of slot 0 sits behind the ring.  The ring length is a multiple of 32
// words, which makes bank(L) = (pitch L + 1 - L + k + TC t) mod 32 injective over the lanes for the pitches used.
template <int TC, int LA> struct SmGeo {
    static constexpr int NT = LA + 1 + (31 + TC - 1) / TC;
    static constexpr int NB = LA + 1;                        // mbarriers
    static constexpr int RING = NT * TC;                     // words
    static constexpr int PITCH = RING + TC;                  // words
    static constexpr int TILE_BYTES = 32 * PITCH * 4;        // rows 0..31 (row 0 = the virtual row above, stays zero)
    static_assert(RING % 32 == 0, "ring must be a multiple of 32 words (bank-conflict-free reads)");
    static_assert(16 % TC == 0 || TC % 16 == 0, "tile must divide or be a multiple of a direction word");
    static constexpr int warp_bytes(bool dirs_smem) { return TILE_BYTES + (dirs_smem ? DS_WORDS * 32 * 4 : 0) + 64; }
};

// float32 -> float64 widening on the INTEGER pipe (exact for zeros and normal numbers; `ok` = false for denormals, inf and
// nan, which the caller widens with the fp64-pipe conversion instead).  Experiment WTS_DTW_VARIANT=5: takes one of the four
// fp64-pipe instructions of an anti-diagonal step (3 DADD + 1 F2F) off that pipe.
__device__ __forceinline__ double widen_f32_int(uint32_t u, bool& ok)
{
    const uint32_t mag = u & 0x7fffffffu;
    const uint32_t e = mag >> 23;
    ok = (e != 255u) && (e != 0u || mag == 0u);
    const uint32_t hi = (mag == 0u ? 0u : (mag >> 3) + 0x38000000u) | (u & 0x80000000u);
    return __hiloint2double((int)hi, (int)(u << 29));
}

template <int TC, int LA, bool DIRS_SMEM, bool INTW = false>
__global__ void __launch_bounds__(32)
dtw_small_kernel(const float* __restrict__ cost, const WtsSegDesc* __restrict__ segs, const int nseg,
                 uint32_t* __restrict__ dir_ws, int32_t* __restrict__ jumps_out, const int l2_prefetch, const int n_rows,
                 const int n_dir_words)
{
    // n_rows: row buffers in shared memory (1 + the largest T of the batch, <= 32); n_dir_words: direction words per lane
    // (for the largest F of the batch, <= DS_WORDS) — sized per launch so that more warps fit an SM
    using G = SmGeo<TC, LA>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const int lane = threadIdx.x;
    const int seg = blockIdx.x;                              // one warp (= one CTA) per matrix
    if (seg >= nseg) return;
    const WtsSegDesc sd = segs[seg];
    if (!dtw_small_eligible(sd) || sd.T + 1 > n_rows || dtw_wpr(sd.F) > n_dir_words) return;   // the general kernel owns it
    unsigned char* my = smem_raw;
    const uint32_t tile_a = smem_u32(my);
    const int tile_bytes = n_rows * G::PITCH * 4;
    uint32_t* dirs = DIRS_SMEM ? reinterpret_cast<uint32_t*>(my + tile_bytes) : dir_ws + sd.dir_off;

    const int T = sd.T, F = sd.F, P = (F + 3) & ~3;
    const float* C = cost + sd.cost_off;
    // Optional (WTS_DTW_L2PF=1): one bulk L2 prefetch of the whole contiguous matrix (T x P float32, <= 44 KB), so that
    // the 64..128-byte tile copies hit L2.  Off by default: the kernel is bound by its dependent chain, not by the DRAM
    // access pattern.
    if (lane == 0 && l2_prefetch)
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(C), "r"((uint32_t)(T * P * 4)) : "memory");
    // zero the row buffers once: cells read before their tile arrives (j < 0), rows beyond T and the virtual row 0
    // must hold finite values (INF + 0 stays INF; they never feed a cell of the matrix)
    {
        float4* z = reinterpret_cast<float4*>(my);
        for (int k = lane; k < tile_bytes / 16; k += 32) z[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncwarp();

    const int niter = dtw_niter(F);                          // 32-step tiles of the wavefront (direction layout: 2 words each)
    const int nit = niter * (32 / TC);                       // TC-step iterations
    const int ntile = (P + TC - 1) / TC;                     // column tiles of the matrix
    // Staging: 16-byte cp.async (LDGSTS.128).  A lane owns chunk `cq` (4 columns) of the rows rq, rq + RPI, ... of every
    // tile: one warp instruction moves 32 chunks = RPI rows x TC columns, so a tile of T <= 31 rows costs
    // ceil(T / RPI) instructions (twice that when its ring slot is mirrored) plus their address arithmetic.
    // (A per-lane cp.async.bulk looked like "one instruction for all rows" in PTX, but SASS serialises it: ELECT + R2UR +
    // UBLKCP + branch per active lane, ~10 issue slots per copy — 17 of the 39 instructions per step in the ncu capture.)
    constexpr int CPR = TC / 4;                              // 16-byte chunks per row and tile
    constexpr int RPI = 32 / CPR;                            // rows per warp instruction
    constexpr int NG = (31 + RPI - 1) / RPI;                 // instructions per tile
    const int cq = lane % CPR, rq = lane / CPR;
    const float* src_lane = C + (int64_t)rq * P + 4 * cq;
    const uint32_t dst_lane = tile_a + (uint32_t)(rq + 1) * (G::PITCH * 4) + 16u * cq;

    auto issue_tile = [&](int u) {                           // columns [TC u, TC u + TC) of every row -> ring slot u % NT
        if (u < ntile) {
            const int slot = u % G::NT;
            const bool col_ok = TC * u + 4 * cq < P;
#pragma unroll
            for (int g = 0; g < NG; ++g) {
                if (col_ok && rq + RPI * g < T) {
                    const float* src = src_lane + (int64_t)(RPI * g) * P + TC * u;
                    const uint32_t dst = dst_lane + (uint32_t)(RPI * g) * (G::PITCH * 4) + (uint32_t)(slot * TC * 4);
                    cp_async<16>(dst, src);
                    if (slot == 0) cp_async<16>(dst + G::RING * 4, src);      // mirror behind the ring
                }
            }
        }
        cp_async_commit();                                   // one group per tile, also when nothing was issued
    };

    const double INF = dinf();
    double cur = INF, upprev = INF;
    if (lane == 1) upprev = 0.0;                             // seeds cm[0,0] = 0 + lm[0,0]
    uint32_t pb = (uint32_t)((G::RING - lane + 1) % G::RING) * 4u;   // 4 * ((TC t - L + 1) mod RING), t = 0
    uint32_t acc = 0;
    const uint32_t myrow_a = tile_a + min(lane, n_rows - 1) * (G::PITCH * 4);   // lanes beyond the buffers re-read the last row
#pragma unroll
    for (int u = 0; u < LA; ++u) issue_tile(u);
    for (int t = 0; t < nit; ++t) {
        cp_async_wait<LA - 1>();                             // all but the newest LA - 1 groups have landed: tile t is in
        __syncwarp();
        issue_tile(t + LA);                                  // its ring slot held a tile last read in iteration t - 1
        const uint32_t rd = myrow_a + pb;
        const int s0 = (t * TC) & 15;                        // position of this tile inside its direction word
        if (s0 == 0) acc = 0;
#pragma unroll
        for (int k = 0; k < TC; ++k) {
            double l;
            if (INTW) {
                const float lf = lds<float>(rd + 4 * k);
                bool ok;
                l = widen_f32_int(__float_as_uint(lf), ok);
                if (__any_sync(FULL_MASK, !ok)) l = (double)lf;      // denormal / non-finite somewhere in the warp: rare
            } else {
                l = (double)lds<float>(rd + 4 * k);
            }
            const double up = __shfl_up_sync(FULL_MASK, cur, 1);
            const double c1 = upprev + l, c2 = cur + l, c3 = up + l;
            upprev = up;
            // all sums are strictly negative doubles or +inf: a < b  <=>  bits(a) >u bits(b)
            const bool p2 = (unsigned long long)__double_as_longlong(c2) > (unsigned long long)__double_as_longlong(c1);
            const double m = p2 ? c2 : c1;
            const bool p3 = (unsigned long long)__double_as_longlong(c3) > (unsigned long long)__double_as_longlong(m);
            cur = p3 ? c3 : m;
            if (TC >= 16) {
                if ((k & 15) == 0) acc = 0;
                if (p2) acc |= 1u << (2 * (k & 15));
                if (p3) acc |= 2u << (2 * (k & 15));
                if ((k & 15) == 15) dirs[((t * TC + k) >> 4) * 32 + lane] = acc;
            } else {
                if (p2) acc |= (1u << (2 * k)) << (2 * s0);
                if (p3) acc |= (2u << (2 * k)) << (2 * s0);
            }
        }
        if (TC < 16 && s0 + TC == 16) dirs[((t * TC) >> 4) * 32 + lane] = acc;
        pb += TC * 4;
        if (pb >= (uint32_t)(G::RING * 4)) pb -= G::RING * 4;
    }
    cp_async_wait<0>();
    if (!DIRS_SMEM) __threadfence_block();
    __syncwarp();
    dtw_backtrack_jumps(dirs, 2 * niter, T, F, jumps_out + sd.jumps_off, lane);
}

// ------------------------------------------------------------------------------------ lane-per-matrix path (large batches)
// With thousands of matrices in one call the wavefront kernels above are bound by their dependent chain, and that chain
// carries a shuffle per cell (lane = row: `up` comes from the neighbouring lane).  Here a LANE owns a whole matrix
// (T <= TR <= 32 rows, any F) and a warp walks 32 matrices column by column: the column of accumulated costs lives in
// registers (D[TR], statically indexed), `up` is the value the same lane produced one cell earlier, `left` / `diag` are
// the previous column's registers — no shuffle, no shared memory in the recurrence.  Two columns advance together,
// skewed by one row (cell (s, j) and cell (s-1, j+1) in step s), which gives every lane two independent chains to
// interleave.  Same three fp64 sums, same strict compares, same tie-breaks as the kernels above (bit-identical).
//  * staging: the warp copies the next tile (8 columns = one 32-byte sector of every row of its 32 matrices) with
//    16-byte cp.async while it computes the current one: two lanes per sector, 8 rows x 2 matrices per instruction,
//    `.L2::128B` so that DRAM sees 128-byte requests and the following three tiles hit L2.  Shared layout
//    [slot][row][half][matrix] x 16 bytes: a lane's LDS.64 of (row, column pair) is base + immediate.
//  * directions: 2 bits per cell, one word per (16 columns, row), TR words of a column group contiguous per matrix
//    (128-bit stores every 16 columns); the backtrack runs per lane on its own matrix (one step per token row, clz
//    over the packed words), reading back what the same thread wrote.
// Throughput kernel: its latency is that of one matrix walked serially (T F cells), so it only pays when the batch
// fills the machine (wts_dtw_batch_sized picks it from WTS_DTW_LANE_MIN matrices on).

__device__ __forceinline__ void cp_async_cg16_l2(uint32_t dst, const void* src)
{
    asm volatile("cp.async.cg.shared.global.L2::128B [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ float2 lds_f2(uint32_t addr)
{
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ float4 lds_f4(uint32_t addr)
{
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ bool neg_less(double a, double b)   // a < b for strictly negative doubles or +inf
{
    return (unsigned long long)__double_as_longlong(a) > (unsigned long long)__double_as_longlong(b);
}

// one cell: the first strict minimum of (diag, left, up) sums wins; direction bits ORed into the row's word by two
// predicated instructions (written in PTX: the compiler's own choice was SEL + SEL + LOP3)
__device__ __forceinline__ double dtw_lane_cell(const double c1, const double c2, const double c3, uint32_t& acc,
                                                const uint32_t one, const uint32_t two)
{
    unsigned long long cur;
    asm("{\n\t.reg .pred p2, p3;\n\t.reg .b64 m;\n\t"
        "setp.gt.u64 p2, %3, %2;\n\t"          // c2 < c1  (strictly negative doubles or +inf: a < b <=> bits(a) >u bits(b))
        "selp.b64 m, %3, %2, p2;\n\t"
        "setp.gt.u64 p3, %4, m;\n\t"           // c3 < min(c1, c2)
        "selp.b64 %0, %4, m, p3;\n\t"
        "@p2 or.b32 %1, %1, %5;\n\t"
        "@p3 or.b32 %1, %1, %6;\n\t}"
        : "=l"(cur), "+r"(acc)
        : "l"((unsigned long long)__double_as_longlong(c1)), "l"((unsigned long long)__double_as_longlong(c2)),
          "l"((unsigned long long)__double_as_longlong(c3)), "r"(one), "r"(two));
    return __longlong_as_double((long long)cur);
}

template <int TR, int G> struct LaneGeo {
    static constexpr int MPW = 32 / G;                       // matrices per warp
    static constexpr int RL = TR / G;                        // rows per lane (one band of the matrix)
    static constexpr int CHUNK_BYTES = MPW * 16;             // [matrix] x 16 bytes (4 columns)
    static constexpr int ROW_BYTES = 2 * CHUNK_BYTES;        // [half][matrix] x 16 bytes
    static constexpr int SLOT_BYTES = TR * ROW_BYTES;
    static constexpr int TABLE_BYTES = 32 * 16;
    static constexpr int SMEM = TABLE_BYTES + 2 * SLOT_BYTES;
};

// NC adjacent columns j .. j + NC - 1 of one band (RL rows) of every lane's matrix, skewed by one row: in step s chain c
// sits on cell (s - c, j + c), so a lane has NC independent dependent chains to interleave.  Chain c's `left` / `diag`
// are what chain c - 1 produced one / two steps earlier; chain 0 reads the previous column from D, the last chain
// writes D back.  bnd[c]: the accumulated cost just above the band in column j + c (+inf for the first band), diag0:
// the same for column j - 1 (0 for the very first cell); last[c] returns the band's last row.
// D: column j - 1 on entry, column j + NC - 1 on exit.  lv: the band's local costs of the group (dtw_lane_load).
template <int RL, int NC, int ROW_BYTES>
__device__ __forceinline__ void dtw_lane_load(float (&lv)[RL][NC], const uint32_t ld_addr)
{
#pragma unroll
    for (int i = 0; i < RL; ++i) {
        if (NC == 4) {
            const float4 v = lds_f4(ld_addr + i * ROW_BYTES);
            lv[i][0] = v.x; lv[i][1] = v.y; lv[i][NC - 2] = v.z; lv[i][NC - 1] = v.w;
        } else {
            const float2 v = lds_f2(ld_addr + i * ROW_BYTES);
            lv[i][0] = v.x; lv[i][1] = v.y;
        }
    }
}

template <int RL, int NC>
__device__ __forceinline__ void dtw_lane_cols(double (&D)[RL], uint32_t (&acc)[RL], const float (&lv)[RL][NC], const double diag0,
                                              const double (&bnd)[NC], double (&last)[NC], const uint32_t one, const uint32_t two)
{
    static_assert(NC == 2 || NC == 4, "two or four columns per group");
    const double INF = dinf();
    double up[NC], h1[NC], h2[NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) { up[c] = bnd[c]; h1[c] = INF; h2[c] = INF; }
    h1[0] = bnd[0];                                          // chain 0 "at row -1" one step before the first
    double diagA = diag0;
#pragma unroll
    for (int s = 0; s < RL + NC - 1; ++s) {
        double out[NC];
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const int r = s - c;
            if (r < 0 || r >= RL) { out[c] = (r == -1) ? bnd[c] : INF; continue; }
            const double l = (double)lv[r][c];
            const double left = (c == 0) ? D[r] : h1[c > 0 ? c - 1 : 0];
            const double diag = (c == 0) ? diagA : h2[c > 0 ? c - 1 : 0];
            const double cur = dtw_lane_cell(diag + l, left + l, up[c] + l, acc[r], one << (2 * c), two << (2 * c));
            up[c] = cur;
            out[c] = cur;
            if (c == 0) diagA = left;
            if (c == NC - 1) D[r] = cur;
            if (r == RL - 1) last[c] = cur;
        }
#pragma unroll
        for (int c = 0; c < NC; ++c) { h2[c] = h1[c]; h1[c] = out[c]; }
    }
}

// Direction words of the lane path: one word = 16 columns x 2 bits of one row.  They are stored in blocks of
// (2 column groups x 4 rows) = 32 bytes, so that the backtrack — a chain of dependent L2 reads that walks up and to the
// left — finds the neighbouring rows and the previous column group of its position in the sector it already holds.
template <int TR>
__host__ __device__ __forceinline__ int64_t dtw_lane_dir_index(int g16, int row)
{
    return (((int64_t)(g16 >> 1) * (TR / 4) + (row >> 2)) << 3) + ((g16 & 1) << 2) + (row & 3);
}

// G lanes per matrix: lane = band * MPW + matrix, band b owns rows [b RL, (b + 1) RL) and runs b column groups behind
// band b - 1, whose last row it receives by shuffle once per group (not per cell).
template <int TR, int NC, int G>
__global__ void __launch_bounds__(32)
dtw_lane_kernel(const float* __restrict__ cost, const WtsSegDesc* __restrict__ segs, const int nseg,
                uint32_t* dir_ws, int32_t* __restrict__ jumps_out, const int bt_bytes)
{
    // bt_bytes: shared-memory bytes per matrix for the backtrack's copy of the direction words (0 = walk them in L2)
    using Geo = LaneGeo<TR, G>;
    constexpr int MPW = Geo::MPW, RL = Geo::RL, GPT = 8 / NC;   // GPT: column groups per tile
    static_assert(TR % 8 == 0 && TR <= 32 && (G == 1 || G == 2 || G == 4) && TR % G == 0, "rows per matrix: 8, 16, 24 or 32; 1, 2 or 4 bands");
    static_assert(G - 1 < GPT, "the last band must leave a tile before the tile after next is issued into its slot");
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    const int lane = threadIdx.x;
    const int band = lane / MPW, mi = lane % MPW;
    const int seg = blockIdx.x * MPW + mi;                   // one warp (= one CTA) per MPW matrices
    WtsSegDesc sd;
    bool mine = false;
    if (seg < nseg) { sd = segs[seg]; mine = dtw_lane_eligible(sd, TR); }
    const int T = mine ? sd.T : 0, F = mine ? sd.F : 0, P = mine ? ((sd.F + 3) & ~3) : 0;
    const float* C = mine ? cost + sd.cost_off : cost;
    uint4* table = reinterpret_cast<uint4*>(smem_raw);       // per matrix: source pointer, row pitch, rows
    if (band == 0) {
        const unsigned long long a = (unsigned long long)(uintptr_t)C;
        table[mi] = make_uint4((uint32_t)a, (uint32_t)(a >> 32), (uint32_t)P, (uint32_t)T);
    }
    const uint32_t stage_a = smem_u32(smem_raw + Geo::TABLE_BYTES);
    int Fmax = F;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) Fmax = max(Fmax, __shfl_xor_sync(FULL_MASK, Fmax, o));
    if (Fmax == 0) return;                                   // nothing here for this path (the general kernel owns them)
    __syncwarp();
    const int ntile = (Fmax + 7) >> 3;

    // Staging roles: two lanes per 32-byte sector, 8 rows x 2 matrices per warp instruction.  What a lane needs to
    // know about the MPW / 2 matrices it copies for (source of its row / half-sector, pitch, rows) stays in registers,
    // so that issuing a tile is straight-line code with no loads in front of the address arithmetic.
    const int half = lane & 1, rr = (lane >> 1) & 7, mm = lane >> 4;
    const float* sp[MPW / 2];                                // (matrix 2 k + mm, row rr, column 4 half)
    uint32_t sq[MPW / 2];                                    // rows << 16 | pitch
#pragma unroll
    for (int k = 0; k < MPW / 2; ++k) {
        const uint4 d = table[2 * k + mm];
        sp[k] = reinterpret_cast<const float*>((uintptr_t)(((unsigned long long)d.y << 32) | d.x)) + (int64_t)rr * (int)d.z + 4 * half;
        sq[k] = (d.w << 16) | d.z;
    }
    const uint32_t dst_lane = stage_a + (uint32_t)rr * Geo::ROW_BYTES + (uint32_t)half * Geo::CHUNK_BYTES + (uint32_t)mm * 16;
    auto issue_tile = [&](int t) {
        if (t < ntile) {
            const int col = 8 * t + 4 * half;
            const uint32_t dst0 = dst_lane + (uint32_t)(t & 1) * Geo::SLOT_BYTES;
#pragma unroll
            for (int k = 0; k < MPW / 2; ++k) {
                const int Pm = (int)(sq[k] & 0xffffu), Tm = (int)(sq[k] >> 16);
                const bool col_ok = col < Pm;
                const float* src = sp[k] + 8 * t;
#pragma unroll
                for (int rb = 0; rb < TR / 8; ++rb)
                    if (col_ok && rr + 8 * rb < Tm)
                        cp_async_cg16_l2(dst0 + (uint32_t)k * 32 + (uint32_t)rb * 8 * Geo::ROW_BYTES, src + (int64_t)(rb * 8) * Pm);
            }
        }
        cp_async_commit();                                   // one group per tile, also when nothing was issued
    };

    double D[RL];
    uint32_t acc[RL];
    const double INF = dinf();
#pragma unroll
    for (int i = 0; i < RL; ++i) { D[i] = INF; acc[i] = 0; }
    uint32_t* dirs = dir_ws + (mine ? sd.dir_off : 0);       // word of (16-column group g, row i): dtw_lane_dir_index
    const int ngroups16 = (F + 15) >> 4;
    const uint32_t row_a = stage_a + (uint32_t)(band * RL) * Geo::ROW_BYTES + (uint32_t)mi * 16;
    double last[NC], plast = INF;                            // this band's last row: previous group, and its last column before
#pragma unroll
    for (int c = 0; c < NC; ++c) last[c] = INF;

    const int nsteps = ntile * GPT + (G - 1);                // band b handles column group (step - b)
    double nb[NC], nd = INF;                                 // the band above's last row, shuffled at the end of the previous step
#pragma unroll
    for (int c = 0; c < NC; ++c) nb[c] = INF;
    issue_tile(0);
#pragma unroll 1
    for (int gs = 0; gs < nsteps; ++gs) {
        const int t = gs / GPT, p = gs % GPT;
        if (p == 0 && t < ntile) {
            cp_async_wait<0>();                              // tile t has landed (this lane's copies)
            __syncwarp();                                    // ... and everybody's
        }
        const int mg = gs - band;                            // this lane's column group
        const int mgc = max(mg, 0);
        const int j = NC * mgc;
        const int tm = mgc / GPT, pm = mgc % GPT;
        const uint32_t sh = 2u * (uint32_t)(j & 15);
        float lv[RL][NC];                                    // local costs of the group: loaded first, consumed after the copies below
        dtw_lane_load<RL, NC, Geo::ROW_BYTES>(lv, row_a + (uint32_t)(tm & 1) * Geo::SLOT_BYTES +
                                                      (uint32_t)((NC * pm) >> 2) * Geo::CHUNK_BYTES + (uint32_t)((NC * pm) & 3) * 4);
        if (p == G - 1) {
            // the slot of tile t + 1 held tile t - 1, which the last band read until the previous step
            if (G > 1) __syncwarp();
            issue_tile(t + 1);
        }
        double bnd[NC], diag0;
#pragma unroll
        for (int c = 0; c < NC; ++c) bnd[c] = (G == 1 || band == 0) ? INF : nb[c];
        diag0 = (G == 1 || band == 0) ? ((mg == 0) ? 0.0 : INF) : nd;
        plast = last[NC - 1];
        dtw_lane_cols<RL, NC>(D, acc, lv, diag0, bnd, last, 1u << sh, 2u << sh);
        if (G > 1 && mg < 0) {                               // a band that has not started yet: undo the step
#pragma unroll
            for (int i = 0; i < RL; ++i) { D[i] = INF; acc[i] = 0; }
#pragma unroll
            for (int c = 0; c < NC; ++c) last[c] = INF;
            plast = INF;
        }
        if (G > 1) {                                         // hand the last row down for the next step (off its critical path)
#pragma unroll
            for (int c = 0; c < NC; ++c) nb[c] = __shfl_up_sync(FULL_MASK, last[c], MPW);
            nd = __shfl_up_sync(FULL_MASK, plast, MPW);
        }
        if (mg >= 0 && ((j + NC) & 15) == 0) {               // a 16-column direction group is complete
            const int g16 = j >> 4;
            if (g16 < ngroups16) {
                if (RL % 4 == 0) {
#pragma unroll
                    for (int q = 0; q < RL / 4; ++q)
                        *reinterpret_cast<uint4*>(dirs + dtw_lane_dir_index<TR>(g16, band * RL + 4 * q)) =
                            make_uint4(acc[4 * q], acc[4 * q + 1], acc[4 * q + 2], acc[4 * q + 3]);
                } else {
#pragma unroll
                    for (int q = 0; q < RL; ++q) dirs[dtw_lane_dir_index<TR>(g16, band * RL + q)] = acc[q];
                }
            }
#pragma unroll
            for (int i = 0; i < RL; ++i) acc[i] = 0;
        }
    }
    {   // the last, incomplete direction group
        const int jend = NC * (nsteps - band);               // first column this lane has not processed
        if ((jend & 15) != 0) {
            const int g16 = jend >> 4;
            if (g16 < ngroups16) {
#pragma unroll
                for (int q = 0; q < RL; ++q) dirs[dtw_lane_dir_index<TR>(g16, band * RL + q)] = acc[q];
            }
        }
    }
    cp_async_wait<0>();
    __syncwarp();                                            // direction words of all bands are visible to the whole warp

    // The backtrack is a chain of dependent reads.  When the batch's direction words fit the (now idle) staging
    // buffers, the warp first copies them back from L2 in one pipelined sweep and walks them in shared memory.
    const int dir_bytes = ((ngroups16 + 1) >> 1) * (TR / 4) * 32;
    const bool in_smem = bt_bytes > 0 && __all_sync(FULL_MASK, !mine || dir_bytes <= bt_bytes);
    if (in_smem) {
#pragma unroll 1
        for (int m = 0; m < MPW; ++m) {                      // lane m = band 0 of matrix m
            const unsigned long long src = __shfl_sync(FULL_MASK, (unsigned long long)(uintptr_t)dirs, m);
            const int nch = __shfl_sync(FULL_MASK, mine ? dir_bytes >> 4 : 0, m);
            for (int c = lane; c < nch; c += 32)
                cp_async_cg16_l2(stage_a + (uint32_t)(m * bt_bytes + 16 * c), reinterpret_cast<const char*>((uintptr_t)src) + 16 * c);
        }
        cp_async_commit();
        cp_async_wait<0>();
        __syncwarp();
    }
    if (!mine || band != 0) return;

    // backtrack on this lane's matrix: one step per token row (T.py:1648-1652)
    const uint32_t* dm = in_smem ? reinterpret_cast<const uint32_t*>(smem_raw + Geo::TABLE_BYTES + mi * bt_bytes) : dirs;
    int32_t* jumps = jumps_out + sd.jumps_off;
    int i = T - 1, j = F - 1;
    jumps[T] = F - 1;
    uint4 ce = make_uint4(0, 0, 0, 0), co = ce;              // the 32-byte block (2 column groups x 4 rows) the walk is in
    int ck = -1;
    while (i > 0) {
        int g = j >> 4, pos = j & 15, kf = 0;
        uint32_t x = 0;
        while (true) {
            const int key = (g >> 1) * (TR / 4) + (i >> 2);
            if (key != ck) {
                ck = key;
                const uint4* blk = reinterpret_cast<const uint4*>(dm + ((int64_t)key << 3));
                if (in_smem) { ce = blk[0]; co = blk[1]; }
                else { ce = __ldcg(blk); co = __ldcg(blk + 1); }
            }
            const uint4 cw = (g & 1) ? co : ce;
            x = (i & 2) ? ((i & 1) ? cw.w : cw.z) : ((i & 1) ? cw.y : cw.x);
            const uint32_t msk = dtw_nonleft_mask(x) & (0xffffffffu >> (30 - 2 * pos));
            if (msk) { kf = (31 - __clz(msk)) >> 1; break; }
            if (g == 0) { kf = 0; break; }
            --g; pos = 15;
        }
        const int jj = g * 16 + kf;
        const bool is_up = (x >> (2 * kf + 1)) & 1u;
        jumps[i] = jj;
        j = (!is_up && jj > 0) ? jj - 1 : jj;
        --i;
    }
    jumps[0] = 0;
}

// status: 1 when the segment's local-cost matrix holds a non-finite value (the situation in which
// the reference's dtw() can end with "No warping path found").
template <typename TIn>
__global__ void dtw_status_kernel(const TIn* __restrict__ cost, const WtsSegDesc* __restrict__ segs,
                                  const int nseg, int32_t* __restrict__ status)
{
    const int seg = blockIdx.x;
    if (seg >= nseg) return;
    const WtsSegDesc sd = segs[seg];
    const TIn* C = cost + sd.cost_off;
    const int64_t n = (int64_t)sd.T * seg_pitch(sd);       // padding columns hold zeros (finite)
    int bad = 0;
    for (int64_t k = threadIdx.x; k < n; k += blockDim.x) bad |= !isfinite((double)C[k]);
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) status[seg] = bad ? 1 : 0;
}

}  // namespace wts

using namespace wts;

extern "C" int64_t wts_dtw_dir_words(int32_t T, int32_t F)
{
    if (T <= 0 || F <= 0) return 0;
    return (int64_t)dtw_nstrips(T) * dtw_wpr(F) * 32;
}

extern "C" int64_t wts_dtw_bnd_doubles(int32_t T, int32_t F)
{
    if (T <= RS || F <= 0) return 0;
    return ((int64_t)F + 3) & ~3LL;
}

extern "C" int wts_dtw_batch_sized(const void* d_cost, int32_t cost_is_f64, const WtsSegDesc* d_segs,
                                   int32_t nseg, uint32_t* d_dir_ws, double* d_bnd_ws, int32_t* d_jumps,
                                   int32_t* d_path, const int64_t* d_path_off, int32_t* d_path_len,
                                   int32_t* d_status, int32_t max_T, int32_t max_F, int32_t all_flags, void* stream);

extern "C" int wts_dtw_batch(const void* d_cost, int32_t cost_is_f64, const WtsSegDesc* d_segs,
                             int32_t nseg, uint32_t* d_dir_ws, double* d_bnd_ws, int32_t* d_jumps,
                             int32_t* d_path, const int64_t* d_path_off, int32_t* d_path_len,
                             int32_t* d_status, void* stream)
{
    return wts_dtw_batch_sized(d_cost, cost_is_f64, d_segs, nseg, d_dir_ws, d_bnd_ws, d_jumps, d_path, d_path_off, d_path_len,
                               d_status, 0, 0, 0, stream);
}

extern "C" int wts_dtw_batch_sized(const void* d_cost, int32_t cost_is_f64, const WtsSegDesc* d_segs,
                                   int32_t nseg, uint32_t* d_dir_ws, double* d_bnd_ws, int32_t* d_jumps,
                                   int32_t* d_path, const int64_t* d_path_off, int32_t* d_path_len,
                                   int32_t* d_status, int32_t max_T, int32_t max_F, int32_t all_flags, void* stream)
{
    // max_T / max_F: largest T / F of the batch when the caller knows them (0 = unknown): they size the shared-memory
    // buffers of the single-strip fast path (fewer rows / direction words -> more resident warps)
    const int n_rows = (max_T > 0 && max_T < RS) ? max_T + 1 : RS + 1;
    const int n_dir_words = (max_F > 0 && dtw_wpr(max_F) < DS_WORDS) ? dtw_wpr(max_F) : DS_WORDS;
    if (nseg <= 0) return 0;
    if (!d_cost || !d_segs || !d_dir_ws || !d_jumps) { set_error("wts_dtw_batch: null pointer"); return -2; }
    if (d_path && (!d_path_off || !d_path_len)) { set_error("wts_dtw_batch: d_path needs d_path_off and d_path_len"); return -2; }
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = (nseg + DTW_WARPS - 1) / DTW_WARPS;
    if (cost_is_f64) {
        const size_t smem = (size_t)DTW_WARPS * (TILE_WORDS * sizeof(double) + DS_WORDS * 32 * sizeof(uint32_t));
        WTS_CUDA_CHECK(cudaFuncSetAttribute(dtw_warp_kernel<double>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        dtw_warp_kernel<double><<<grid, DTW_WARPS * 32, smem, st>>>(
            (const double*)d_cost, d_segs, nseg, d_dir_ws, d_bnd_ws, d_jumps, d_path, d_path_off, d_path_len, 0);
        WTS_LAUNCH_CHECK();
        if (d_status) { dtw_status_kernel<double><<<nseg, 128, 0, st>>>((const double*)d_cost, d_segs, nseg, d_status); WTS_LAUNCH_CHECK(); }
    } else {
        // single-strip fast path (dtw_small_kernel) for the segments that qualify; it produces jumps only, so a
        // request for full paths keeps everything in the general kernel.  WTS_DTW_SMALL=0 turns it off.
        // From WTS_DTW_LANE_MIN matrices on (default 8192; 0 = never) the lane-per-matrix kernel takes them instead.
        static const int small_on = [] { const char* e = getenv("WTS_DTW_SMALL"); return e ? atoi(e) : 1; }();
        const char* lane_env = getenv("WTS_DTW_LANE_MIN");  // read per call: tests and benchmarks switch paths at run time
        const int lane_min = lane_env ? atoi(lane_env) : 8192;
        const int use_lane = d_path == nullptr && lane_min > 0 && nseg >= lane_min;
        const int use_small = !use_lane && small_on && d_path == nullptr;
        const int lane_rows = (max_T <= 0 || max_T > 24) ? 32 : max_T > 16 ? 24 : max_T > 8 ? 16 : 8;
        // all_flags (AND of the batch's WtsSegDesc.flags, 0 = unknown) together with the size hints tells when every
        // segment belongs to the fast kernel: the general kernel (whose warps would all exit) is then not launched
        const bool uniform = (all_flags & (WTS_SEG_NONPOSITIVE | WTS_SEG_PITCH16)) == (WTS_SEG_NONPOSITIVE | WTS_SEG_PITCH16) && max_T > 0;
        const bool general_idle = uniform && ((use_lane && max_T <= 32) ||
                                              (use_small && max_T <= RS && max_F > 0 && dtw_wpr(max_F) <= DS_WORDS));
        if (!general_idle) {
            const size_t smem = (size_t)DTW_WARPS * (TILE_WORDS * sizeof(float) + DS_WORDS * 32 * sizeof(uint32_t));
            WTS_CUDA_CHECK(cudaFuncSetAttribute(dtw_warp_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            dtw_warp_kernel<float><<<grid, DTW_WARPS * 32, smem, st>>>(
                (const float*)d_cost, d_segs, nseg, d_dir_ws, d_bnd_ws, d_jumps, d_path, d_path_off, d_path_len,
                use_lane ? (lane_rows << 16) : use_small ? ((n_rows << 8) | n_dir_words) : 0);
            WTS_LAUNCH_CHECK();
        }
        if (use_lane) {
#define WTS_LAUNCH_LANE(TR_, NC_, G_)                                                                                     \
            do {                                                                                                          \
                constexpr int mpw = LaneGeo<TR_, G_>::MPW;                                                                \
                const int warps = (nseg + mpw - 1) / mpw, per_sm = (warps + n_sm - 1) / n_sm;                             \
                /* shared memory a warp may take without lowering the number of resident warps the batch needs */        \
                const int room = per_sm > 0 ? ((232448 / per_sm - 1024) & ~127) : 0;                                      \
                int smem_l = (int)LaneGeo<TR_, G_>::SMEM, bt = 0;                                                         \
                if (max_F > 0 && bt_smem) {                                                                               \
                    const int need = (((max_F + 15) / 16 + 1) / 2) * (TR_ / 4) * 32;                                      \
                    const int tot = (int)LaneGeo<TR_, G_>::TABLE_BYTES + mpw * need;                                      \
                    if (tot <= 232448 - 1024 && (tot <= smem_l || tot <= room)) { bt = need; if (tot > smem_l) smem_l = tot; } \
                }                                                                                                         \
                WTS_CUDA_CHECK(cudaFuncSetAttribute(dtw_lane_kernel<TR_, NC_, G_>,                                        \
                                                    cudaFuncAttributeMaxDynamicSharedMemorySize, smem_l));                \
                dtw_lane_kernel<TR_, NC_, G_><<<warps, 32, smem_l, st>>>((const float*)d_cost, d_segs, nseg, d_dir_ws,    \
                                                                         d_jumps, bt);                                    \
            } while (0)
            static int n_sm = 0;
            if (n_sm == 0) {
                int dev = 0;
                WTS_CUDA_CHECK(cudaGetDevice(&dev));
                WTS_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
            }
            const char* bt_env = getenv("WTS_DTW_LANE_BT_SMEM");   // 0: the backtrack walks the direction words in L2
            const int bt_smem = bt_env ? atoi(bt_env) : 1;
            // WTS_DTW_LANE_NC: columns advanced together per lane (2 or 4 independent chains); WTS_DTW_LANE_G: lanes
            // (row bands) per matrix, 1, 2 or 4 — more bands = more warps per scheduler for the same work
            const char* nc_env = getenv("WTS_DTW_LANE_NC");
            const char* g_env = getenv("WTS_DTW_LANE_G");
            const int lane_g = g_env ? atoi(g_env) : 2;
            const int lane_nc = lane_g == 4 ? 2 : (nc_env && atoi(nc_env) == 2) ? 2 : 4;
#define WTS_LANE_CASE(TR_)                                                                                                \
            if (lane_rows == TR_) {                                                                                       \
                if (lane_g == 1)      { if (lane_nc == 2) WTS_LAUNCH_LANE(TR_, 2, 1); else WTS_LAUNCH_LANE(TR_, 4, 1); }  \
                else if (lane_g == 4) { WTS_LAUNCH_LANE(TR_, 2, 4); }                                                     \
                else                  { if (lane_nc == 2) WTS_LAUNCH_LANE(TR_, 2, 2); else WTS_LAUNCH_LANE(TR_, 4, 2); }  \
            }
            WTS_LANE_CASE(8) WTS_LANE_CASE(16) WTS_LANE_CASE(24) WTS_LANE_CASE(32)
#undef WTS_LANE_CASE
#undef WTS_LAUNCH_LANE
            WTS_LAUNCH_CHECK();
        }
        if (use_small) {
            // geometry variants (WTS_DTW_VARIANT, default 0): <columns per tile, tiles in flight, directions in shared memory>
            static const int variant = [] { const char* e = getenv("WTS_DTW_VARIANT"); return e ? atoi(e) : 4; }();
            static const int l2pf = [] { const char* e = getenv("WTS_DTW_L2PF"); return e ? atoi(e) : 0; }();
#define WTS_LAUNCH_SMALL(TC_, LA_, DS_, IW_)                                                                              \
            do {                                                                                                          \
                const size_t smem_s = (size_t)n_rows * SmGeo<TC_, LA_>::PITCH * 4 + (DS_ ? n_dir_words * 32 * 4 : 0) + 64;      \
                WTS_CUDA_CHECK(cudaFuncSetAttribute(dtw_small_kernel<TC_, LA_, DS_, IW_>,                                 \
                                                    cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_s));          \
                dtw_small_kernel<TC_, LA_, DS_, IW_><<<nseg, 32, smem_s, st>>>((const float*)d_cost, d_segs, nseg,       \
                                                                              d_dir_ws, d_jumps, l2pf, n_rows,           \
                                                                              n_dir_words);                              \
            } while (0)
            switch (variant) {
                case 1: WTS_LAUNCH_SMALL(16, 1, false, false); break;
                case 2: WTS_LAUNCH_SMALL(8, 3, true, false); break;
                case 3: WTS_LAUNCH_SMALL(8, 3, false, false); break;
                case 4: WTS_LAUNCH_SMALL(32, 1, true, false); break;
                case 5: WTS_LAUNCH_SMALL(16, 1, false, true); break;
                case 0: WTS_LAUNCH_SMALL(16, 1, true, false); break;
                default: WTS_LAUNCH_SMALL(32, 1, true, false); break;
            }
#undef WTS_LAUNCH_SMALL
            WTS_LAUNCH_CHECK();
        }
        if (d_status) { dtw_status_kernel<float><<<nseg, 128, 0, st>>>((const float*)d_cost, d_segs, nseg, d_status); WTS_LAUNCH_CHECK(); }
    }
    return 0;
}
