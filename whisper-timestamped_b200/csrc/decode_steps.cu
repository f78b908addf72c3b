// Persistent decode-step kernel for SMALL active batches (<= 32 windows still decoding).
//
// Why: a decoder step of large-v3 is ~355 dependent kernels when every operator is its own launch; at <= 32 active
// windows each of them sits at its launch + prologue floor, far above the time the step's weight stream needs
// from HBM.  Here ONE cooperative kernel (one CTA per SM, all co-resident) walks
//     embed -> L x [LN+QKV | self-attn | out-proj | LN+Q | cross-attn | out-proj | LN+FC1+GELU | FC2] -> LN+logits -> select
// for up to `n_steps` tokens, phases separated by a grid-wide barrier (one atomic + one polling thread per CTA).
// Replaces, for the whole batch at once, upstream's DecodingTask._main_loop step + the reference's per-token hooks
// (T.py:783-793 hook_attention_weights, 849-881 hook_output_logits).
//
// At <= 32 rows the GEMMs are weight-streaming matrix-vector products, so they run on the FP32 pipe (no tensor cores:
// a 128-row tensor-core tile would be >= 75 % padding, and its tensor-map/barrier prologue costs a kernel that
// short more than its math): a warp owns 4 output features, streams their float32 weight rows once (coalesced 512-byte loads, L1
// bypassed), multiplies them with up to 16 activation rows staged in shared memory (LayerNorm fused into the
// staging), and reduces over the lanes with a transposing butterfly that leaves every lane with its own outputs.
// Weights of the NEXT phase are prefetched into L2 before each barrier, so HBM keeps streaming while CTAs wait.
// Results are float32 throughout (weights float32 = the exact values the SB16 tensor-core path carries as hi + lo).
#include "decode_common.cuh"

namespace wts {

constexpr int MG_THREADS = 256;
constexpr int MG_WARPS = MG_THREADS / 32;
constexpr int MG_MAXROWS = 32;          // active rows the staging buffer holds
constexpr int MG_G = 4;                 // output features per warp task
constexpr int MG_MAXNI = 10;            // D / 128 <= 10 (D <= 1280)

struct MgShared {
    int list[MG_MAXROWS];               // active slots, ascending
    int n_active;
    int abort_flag;
    int prof_idx;                       // next slot of the optional phase timeline (block 0 only)
    unsigned long long* prof;
    int prof_cap;
    SelectScratch sel;
};

__device__ __forceinline__ float4 ldg_stream4(const float* p)
{
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// ---- grid-wide barrier.  Arrivals are one release-add per CTA on a counter; the LAST arriver publishes the new
// generation on a different 128-byte line, which is the only thing the other CTAs poll (acquire loads with a short
// back-off) — polls never contend with the arriving atomics (polling the counter itself, or a flag array where every
// CTA publishes its generation and warp 0 polls all of them, both keep the arrivals waiting on the polls).  sync[0] = arrivals, sync[1] = error flag, sync[2] = steps completed, sync[32] = generation.
// A spin limit turns a would-be hang (a bug, or a grid that is not co-resident) into an error flag the host reports.
__device__ __forceinline__ void grid_sync(uint32_t* sync, uint32_t& gen, MgShared& sh)
{
    __syncthreads();
    gen += 1;
    if (threadIdx.x == 0 && !sh.abort_flag) {
        __threadfence();
        uint32_t old;
        asm volatile("atom.add.release.gpu.global.u32 %0, [%1], 1;" : "=r"(old) : "l"(sync) : "memory");
        if (old + 1 == gen * gridDim.x) {
            asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(sync + 32), "r"(gen) : "memory");
        } else {
            uint32_t g;
            int spins = 0;
            while (true) {
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(g) : "l"(sync + 32) : "memory");
                if (g >= gen) break;
                __nanosleep(20);
                if ((++spins & 1023) == 0) {
                    uint32_t e;
                    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(e) : "l"(sync + 1) : "memory");
                    if (e != 0 || spins > (1 << 22)) {       // ~1 s of polling: a bug, or a grid that is not co-resident
                        atomicExch(sync + 1, 1u);
                        sh.abort_flag = 1;
                        break;
                    }
                }
            }
        }
        __threadfence();
    }
    if (threadIdx.x == 0 && sh.prof != nullptr && sh.prof_idx < sh.prof_cap) {   // phase timeline (probe runs only)
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        sh.prof[sh.prof_idx++] = t;
    }
    __syncthreads();
}

// ---- transposing warp reduction: v[i] (i < NV) summed over the 32 lanes; afterwards lane l holds in v[0 .. NV/32)
// the totals of logical indices l * (NV / 32) + j  (NV >= 32), or for NV = 16 in v[0] the total of index l >> 1.
template <int N, int MASK>
__device__ __forceinline__ void treduce_step(float* v, int lane)
{
    if constexpr (N > 1 && MASK >= 1) {
        const bool up = (lane & MASK) != 0;
#pragma unroll
        for (int i = 0; i < N / 2; ++i) {
            const float keep = up ? v[i + N / 2] : v[i];
            const float send = up ? v[i] : v[i + N / 2];
            v[i] = keep + __shfl_xor_sync(FULL_MASK, send, MASK);
        }
        treduce_step<N / 2, MASK / 2>(v, lane);
    } else if constexpr (MASK >= 1) {
        v[0] += __shfl_xor_sync(FULL_MASK, v[0], MASK);
        treduce_step<1, MASK / 2>(v, lane);
    }
}

// ---- staging of activation rows into shared memory (optionally LayerNorm'ed).  Warp w takes rows w, w + 8, ... of the
// pass: all of its 16-byte cp.async.cg copies are issued back to back (one memory round trip for the whole staging;
// .cg = through L2, the rows were produced by other SMs earlier in this launch), then it normalises its own rows in
// place.  xs row r (pitch `ncols`) <- src[list[row_first + r], col0 .. col0 + ncols).  Ends with a CTA barrier.
constexpr int MG_STAGE_FLOATS = MG_MAXROWS * 128 * MG_MAXNI;     // staging capacity: 32 rows x 1280 columns

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

template <bool LN>
__device__ __forceinline__ void stage_rows(const float* src, int64_t ld, int col0, int ncols, int row_first, int nrows,
                                           const float* __restrict__ gam, const float* __restrict__ bet, const MgShared& sh,
                                           float* xs)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c4n = ncols >> 2;
    const uint32_t xs_a = (uint32_t)__cvta_generic_to_shared(xs);
    for (int r = warp; r < nrows; r += MG_WARPS) {
        const float* g = src + (int64_t)sh.list[row_first + r] * ld + col0;
        const uint32_t d = xs_a + (uint32_t)(r * ncols) * 4u;
        for (int c4 = lane; c4 < c4n; c4 += 32) cp_async16(d + 16u * c4, g + 4 * c4);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();
    if (LN) {                                                // ncols == D: the whole row is here
        const int NI = ncols >> 7;
        for (int r = warp; r < nrows; r += MG_WARPS) {
            float4* row = reinterpret_cast<float4*>(xs + (int64_t)r * ncols);
            float4 v[MG_MAXNI];
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < MG_MAXNI; ++k)
                if (k < NI) { v[k] = row[lane + 32 * k]; s += (v[k].x + v[k].y) + (v[k].z + v[k].w); }
            const float mean = warp_sum(s) / (float)ncols;
            float q = 0.f;
#pragma unroll
            for (int k = 0; k < MG_MAXNI; ++k)
                if (k < NI) {
                    const float a = v[k].x - mean, b = v[k].y - mean, c = v[k].z - mean, d = v[k].w - mean;
                    q += (a * a + b * b) + (c * c + d * d);
                }
            const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)ncols + 1e-5f);
#pragma unroll
            for (int k = 0; k < MG_MAXNI; ++k)
                if (k < NI) {
                    const float4 g = __ldg(reinterpret_cast<const float4*>(gam) + lane + 32 * k);
                    const float4 b = __ldg(reinterpret_cast<const float4*>(bet) + lane + 32 * k);
                    v[k].x = (v[k].x - mean) * rstd * g.x + b.x;
                    v[k].y = (v[k].y - mean) * rstd * g.y + b.y;
                    v[k].z = (v[k].z - mean) * rstd * g.z + b.z;
                    v[k].w = (v[k].w - mean) * rstd * g.w + b.w;
                    row[lane + 32 * k] = v[k];
                }
        }
    }
    __syncthreads();
}

// ---- one K chunk (NI * 128 columns) of a warp task: acc[g][b] += W[n0 + g, kc0 ...] . xs[b, ...]
// The weight slices (4 features x one float4 per lane) run through a 4-slot register ring: three slices are always in
// flight while the fourth is multiplied with the staged rows (RB shared-memory float4 loads, 16 FMAs each).
template <int RB>
__device__ __forceinline__ void gemv_slice(const float4 (&w)[MG_G], const float* xp, int pitch, float (&acc)[MG_G * RB])
{
    constexpr int HB = RB > 8 ? 4 : RB;                      // rows per batch of shared-memory loads (bounds live registers)
#pragma unroll
    for (int b0 = 0; b0 < RB; b0 += HB) {
        float4 xv[HB];
#pragma unroll
        for (int b = 0; b < HB; ++b) xv[b] = *reinterpret_cast<const float4*>(xp + (b0 + b) * pitch);
#pragma unroll
        for (int b = 0; b < HB; ++b) {
#pragma unroll
            for (int g = 0; g < MG_G; ++g) {
                float a = acc[g * RB + b0 + b];
                a = fmaf(w[g].x, xv[b].x, a);
                a = fmaf(w[g].y, xv[b].y, a);
                a = fmaf(w[g].z, xv[b].z, a);
                a = fmaf(w[g].w, xv[b].w, a);
                acc[g * RB + b0 + b] = a;
            }
        }
        asm volatile("" ::: "memory");                       // keep the next batch of loads behind this batch's FMAs
    }
}

template <int RB>
__device__ __forceinline__ void gemv_chunk(const float* __restrict__ W, int64_t ldw, int n0, int N, int kc0, int NI,
                                           const float* xs, int pitch, float (&acc)[MG_G * RB])
{
    const int lane = threadIdx.x & 31;
    const float* wp[MG_G];
#pragma unroll
    for (int g = 0; g < MG_G; ++g) wp[g] = W + (int64_t)min(n0 + g, N - 1) * ldw + kc0 + 4 * lane;
    float4 w[4][MG_G];
#pragma unroll
    for (int u = 0; u < 3; ++u)
        if (u < NI) {
#pragma unroll
            for (int g = 0; g < MG_G; ++g) w[u][g] = ldg_stream4(wp[g] + 128 * u);
        }
#pragma unroll 1
    for (int i0 = 0; i0 < NI; i0 += 4) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int i = i0 + u;
            if (i + 3 < NI) {
#pragma unroll
                for (int g = 0; g < MG_G; ++g) w[(u + 3) & 3][g] = ldg_stream4(wp[g] + 128 * (i + 3));
            }
            if (i < NI) gemv_slice<RB>(w[u], xs + 4 * (lane + 32 * i), pitch, acc);
        }
    }
}

enum { EPI_STORE = 0, EPI_ADD = 1, EPI_GELU = 2 };

// ---- epilogue of a warp task after the transposing reduction
template <int RB>
__device__ __forceinline__ void gemv_epilogue(float (&acc)[MG_G * RB], int n0, int N, int row0, const MgShared& sh,
                                              const float* __restrict__ bias, float* out, int64_t ldo, int epi)
{
    const int lane = threadIdx.x & 31;
    constexpr int NV = MG_G * RB;
    treduce_step<NV, 16>(acc, lane);
    constexpr int PER = NV >= 32 ? NV / 32 : 1;
    const int base = NV >= 32 ? lane * PER : lane / (32 / (NV < 32 ? NV : 32));
    const bool writer = NV >= 32 ? true : (lane % (32 / (NV < 32 ? NV : 32))) == 0;
    if (!writer) return;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
        const int idx = base + j;
        const int g = idx / RB, b = idx % RB;
        const int n = n0 + g;
        const int ri = row0 + b;
        if (n < N && ri < sh.n_active) {
            float t = acc[j] + (bias != nullptr ? __ldg(bias + n) : 0.f);
            float* dst = out + (int64_t)sh.list[ri] * ldo + n;
            if (epi == EPI_GELU) t = gelu_erf(t);
            else if (epi == EPI_ADD) t += __ldcg(dst);
            *dst = t;
        }
    }
}

// ---- a whole matrix-vector phase: out[row, n] = epi(sum_k W[n, k] * act[row, k] + bias[n]) for the active rows.
// act rows come from `src` (global, K columns) staged chunk by chunk (D columns each) into shared memory, with
// LayerNorm(gam, bet) fused when LN (then K == D).  Tasks (4 features) are dealt round-robin to the warps of the grid.
template <int RB, bool LN>
__device__ __noinline__ void gemv_phase(const float* __restrict__ W, int N, int K, int D, const float* __restrict__ bias,
                                           const float* src, int64_t lds, const float* gam, const float* bet, float* out,
                                           int64_t ldo, int epi, const MgShared& sh, float* xs)
{
    const int warp = threadIdx.x >> 5;
    const int total_warps = gridDim.x * MG_WARPS;
    const int gw = warp * gridDim.x + blockIdx.x;            // consecutive tasks land on different SMs
    const int nA = sh.n_active;
    const int ntasks = (N + MG_G - 1) / MG_G;
    const int rounds = (ntasks + total_warps - 1) / total_warps;
    const int npass = (nA + RB - 1) / RB;
    // Either every pass's RB rows with all K columns fit the staging buffer (always when K == D): staged ONCE for all
    // rounds and passes.  Or (FC2 with more than 8 active rows) each pass stages its own rows in chunks of Kc columns.
    const bool once = npass * RB * K <= MG_STAGE_FLOATS;     // a pass reads RB rows of the buffer whatever nA is
    const int Kc = once ? K : (MG_STAGE_FLOATS / (RB * D)) * D;
    const int nchunks = (K + Kc - 1) / Kc;
    if (once) stage_rows<LN>(src, lds, 0, K, 0, nA, gam, bet, sh, xs);
    for (int rd = 0; rd < rounds; ++rd) {
        const int t = gw + rd * total_warps;
        const bool has = t < ntasks;
        for (int ps = 0; ps < npass; ++ps) {
            float acc[MG_G * RB];
#pragma unroll
            for (int i = 0; i < MG_G * RB; ++i) acc[i] = 0.f;
            for (int c = 0; c < nchunks; ++c) {
                const int kc = min(Kc, K - c * Kc);
                if (!once) {
                    __syncthreads();                         // previous chunk fully consumed
                    stage_rows<false>(src, lds, c * Kc, kc, ps * RB, min(RB, nA - ps * RB), nullptr, nullptr, sh, xs);
                }
                if (has) gemv_chunk<RB>(W, K, t * MG_G, N, c * Kc, kc >> 7, once ? xs + (int64_t)ps * RB * K : xs, kc, acc);
            }
            if (has) gemv_epilogue<RB>(acc, t * MG_G, N, ps * RB, sh, bias, out, ldo, epi);
        }
    }
}

// L2 prefetch of the weight rows this warp will stream in a later phase
__device__ __forceinline__ void prefetch_phase(const float* W, int N, int K, int max_rounds = 1 << 30)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int total_warps = gridDim.x * MG_WARPS;
    const int gw = warp * gridDim.x + blockIdx.x;
    const int ntasks = (N + MG_G - 1) / MG_G;
    const int lines_per_row = K / 32;                        // 128-byte lines
    for (int t = gw, r = 0; t < ntasks && r < max_rounds; t += total_warps, ++r) {
        for (int ln = lane; ln < MG_G * lines_per_row; ln += 32) {
            const int g = ln / lines_per_row, c = ln - g * lines_per_row;
            const int n = min(t * MG_G + g, N - 1);
            prefetch_l2(W + (int64_t)n * K + c * 32);
        }
    }
}

// At most this many active rows get their cross-attention K/V prefetched into L2 (a "few rows" step leaves HBM idle
// during its matrix-vector phases).  The launcher lowers the cap further so that one layer's prefetched fp16 K + V fit
// in half of the device's L2 (the other half keeps the weight rows the phases stream): large-v3 holds 7.7 MB per row,
// so a 50 MB L2 takes 3 rows.
constexpr int MG_KV_PREFETCH_ROWS = 8;

__device__ __forceinline__ void prefetch_cross_kv(const WtsDecodeSteps& P, const WtsDecLayer& Lr, const MgShared& sh)
{
    const int64_t per_row = (int64_t)P.H * P.n_audio_ctx * 64 * 2;             // bytes of fp16 K (and of V) per row
    const int64_t lines_row = per_row / 128;
    const int64_t nthreads = (int64_t)gridDim.x * MG_THREADS, me = (int64_t)blockIdx.x * MG_THREADS + threadIdx.x;
    for (int i = 0; i < sh.n_active; ++i) {
        const char* k = reinterpret_cast<const char*>(Lr.cross_k16) + (int64_t)sh.list[i] * per_row;
        const char* v = reinterpret_cast<const char*>(Lr.cross_v16) + (int64_t)sh.list[i] * per_row;
        for (int64_t ln = me; ln < lines_row; ln += nthreads) {
            prefetch_l2(k + ln * 128);
            prefetch_l2(v + ln * 128);
        }
        // float32 K of the alignment heads of this layer
        const int64_t al_row = (int64_t)P.n_slots * P.n_audio_ctx * 64 * 4;
        const char* ka = reinterpret_cast<const char*>(Lr.cross_k_align) + (int64_t)sh.list[i] * al_row;
        for (int h = 0; h < P.H; ++h) {
            const int slot = __ldg(Lr.head_slot + h);
            if (slot < 0) continue;
            const int64_t lines = (int64_t)P.n_audio_ctx * 64 * 4 / 128;
            for (int64_t ln = me; ln < lines; ln += nthreads) prefetch_l2(ka + (int64_t)slot * lines * 128 + ln * 128);
        }
    }
}

// ---- causal self-attention of ONE (row, head) by a warp; appends this position's K/V to the cache first.
// `sc`: this warp's shared-memory scratch, n_ctx floats (scores, then probabilities).
__device__ __noinline__ void self_attention_task(const WtsDecodeSteps& P, const WtsDecLayer& Lr, int row, int h, int pos,
                                                    float* sc)
{
    const int lane = threadIdx.x & 31;
    const int D = P.D, n_ctx = P.n_ctx;
    float* Kc = Lr.self_k + ((int64_t)row * P.H + h) * n_ctx * 64;
    float* Vc = Lr.self_v + ((int64_t)row * P.H + h) * n_ctx * 64;
    const float* qrow = P.qkv + (int64_t)row * 3 * D + h * 64;
    {   // append (float2 per lane), then make it visible to the lanes that read it back below
        const float2 kn = __ldcg(reinterpret_cast<const float2*>(qrow + D) + lane);
        const float2 vn = __ldcg(reinterpret_cast<const float2*>(qrow + 2 * D) + lane);
        reinterpret_cast<float2*>(Kc + (int64_t)pos * 64)[lane] = kn;
        reinterpret_cast<float2*>(Vc + (int64_t)pos * 64)[lane] = vn;
        __threadfence_block();
        __syncwarp();
    }
    float q[64];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
        const float4 t = ldcg4(qrow + 4 * c);
        q[4 * c] = t.x; q[4 * c + 1] = t.y; q[4 * c + 2] = t.z; q[4 * c + 3] = t.w;
    }
    const int nk = pos + 1;
    float mx = -CUDART_INF_F;
#pragma unroll 1
    for (int j = lane; j < nk; j += 32) {                    // a lane owns keys lane, lane + 32, ...
        const float* kr = Kc + (int64_t)j * 64;
        float a = 0.f;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            const float4 kv = ldcg4(kr + 4 * c);
            a += q[4 * c] * kv.x + q[4 * c + 1] * kv.y + q[4 * c + 2] * kv.z + q[4 * c + 3] * kv.w;
        }
        sc[j] = a;
        mx = fmaxf(mx, a);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll 1
    for (int j = lane; j < nk; j += 32) {
        const float e = expf(sc[j] - mx);
        sc[j] = e;
        sum += e;
    }
    sum = warp_sum(sum);
    __syncwarp();
    float2 o = make_float2(0.f, 0.f);                        // a lane owns channels 2 lane, 2 lane + 1
#pragma unroll 8
    for (int j = 0; j < nk; ++j) {
        const float p = sc[j];
        const float2 v = __ldcg(reinterpret_cast<const float2*>(Vc + (int64_t)j * 64) + lane);
        o.x = fmaf(p, v.x, o.x);
        o.y = fmaf(p, v.y, o.y);
    }
    const float inv = 1.0f / sum;
    reinterpret_cast<float2*>(P.att + (int64_t)row * D + h * 64)[lane] = make_float2(o.x * inv, o.y * inv);
    __syncwarp();                                            // scratch is reused by this warp's next task
}

// ---- cross-attention of the active rows: one CTA per (row, head), K/V (fp16; float32 K for the alignment heads) are
// streamed once; the alignment heads' pre-softmax rows go straight into the alignment buffer (qk_buf).
__device__ __noinline__ void cross_attention_phase(const WtsDecodeSteps& P, const WtsDecLayer& Lr, const MgShared& sh, float* xs)
{
    const int D = P.D, H = P.H;
    CaScratch& sc = *reinterpret_cast<CaScratch*>(xs);
    const int c8 = threadIdx.x & 7;
    for (int t = blockIdx.x; t < sh.n_active * H; t += gridDim.x) {
        const int row = sh.list[t / H], h = t % H;
        float qf[8];
        {
            const float* qp = P.q + (int64_t)row * D + h * 64 + c8 * 8;
            const float4 a = ldcg4(qp), b = ldcg4(qp + 4);
            qf[0] = a.x; qf[1] = a.y; qf[2] = a.z; qf[3] = a.w; qf[4] = b.x; qf[5] = b.y; qf[6] = b.z; qf[7] = b.w;
        }
        const int slot = __ldg(Lr.head_slot + h);
        const int64_t kv_off = ((int64_t)row * H + h) * P.n_audio_ctx * 64;
        const float* kal = nullptr;
        float* qk_dst = nullptr;
        if (slot >= 0) {
            kal = Lr.cross_k_align + ((int64_t)row * P.n_slots + slot) * P.n_audio_ctx * 64;
            const int qr = __ldcg(P.n_tokens + row) - __ldg(P.n_prompt + row);
            qk_dst = P.qk_buf + (((int64_t)row * P.n_slots + slot) * P.qk_rows + qr) * (int64_t)P.n_audio_ctx;
        }
        const float y = ca_row_head<4>(qf, reinterpret_cast<const __half*>(Lr.cross_k16) + kv_off,
                                       reinterpret_cast<const __half*>(Lr.cross_v16) + kv_off, kal, qk_dst,
                                       P.n_audio_ctx, sc);
        if (threadIdx.x < 64) P.att[(int64_t)row * D + h * 64 + threadIdx.x] = y;
        __syncthreads();                                     // scratch reused by the next task
    }
}

template <int RB>
__device__ void decode_layers_and_logits(const WtsDecodeSteps& P, MgShared& sh, float* xs, uint32_t& target, int kv_pf_rows)
{
    const int D = P.D, H = P.H;
    const int warp = threadIdx.x >> 5;
    const int total_warps = gridDim.x * MG_WARPS;
    const int gw = warp * gridDim.x + blockIdx.x;
    for (int li = 0; li < P.n_layer; ++li) {
        const WtsDecLayer& Lr = P.layers[li];
        // few active rows: pull this layer's cross-attention K/V into L2 now (the matrix-vector phases in between leave HBM
        // idle), so the (row, head) streams of P5 — each a single CTA with limited bytes in flight — run at L2 latency
        if (sh.n_active <= kv_pf_rows) prefetch_cross_kv(P, Lr, sh);
        // P1: LN + QKV
        gemv_phase<RB, true>(Lr.w_qkv, 3 * D, D, D, Lr.b_qkv, P.x, D, Lr.ln1_g, Lr.ln1_b, P.qkv, 3 * D, EPI_STORE, sh, xs);
        prefetch_phase(Lr.w_o, D, D);
        grid_sync(P.sync, target, sh);
        // P2: self-attention, one warp per (row, head)
        for (int t = gw; t < sh.n_active * H; t += total_warps) {
            const int row = sh.list[t / H];
            self_attention_task(P, Lr, row, t % H, __ldcg(P.n_tokens + row) - 1, xs + warp * P.n_ctx);
        }
        grid_sync(P.sync, target, sh);
        // P3: out-projection + residual
        gemv_phase<RB, false>(Lr.w_o, D, D, D, Lr.b_o, P.att, D, nullptr, nullptr, P.x, D, EPI_ADD, sh, xs);
        prefetch_phase(Lr.w_cq, D, D);
        grid_sync(P.sync, target, sh);
        // P4: LN + cross query
        gemv_phase<RB, true>(Lr.w_cq, D, D, D, Lr.b_cq, P.x, D, Lr.ln2_g, Lr.ln2_b, P.q, D, EPI_STORE, sh, xs);
        prefetch_phase(Lr.w_co, D, D);
        grid_sync(P.sync, target, sh);
        // P5: cross-attention, one CTA per (row, head); scratch aliases the (idle) staging buffer
        cross_attention_phase(P, Lr, sh, xs);
        grid_sync(P.sync, target, sh);
        // P6: cross out-projection + residual
        gemv_phase<RB, false>(Lr.w_co, D, D, D, Lr.b_co, P.att, D, nullptr, nullptr, P.x, D, EPI_ADD, sh, xs);
        prefetch_phase(Lr.w_fc1, 4 * D, D);
        grid_sync(P.sync, target, sh);
        // P7: LN + FC1 + GELU
        gemv_phase<RB, true>(Lr.w_fc1, 4 * D, D, D, Lr.b_fc1, P.x, D, Lr.ln3_g, Lr.ln3_b, P.mid, 4 * D, EPI_GELU, sh, xs);
        prefetch_phase(Lr.w_fc2, D, 4 * D);
        grid_sync(P.sync, target, sh);
        // P8: FC2 + residual (K = 4D in D-column chunks)
        gemv_phase<RB, false>(Lr.w_fc2, D, 4 * D, D, Lr.b_fc2, P.mid, 4 * D, nullptr, nullptr, P.x, D, EPI_ADD, sh, xs);
        if (li + 1 < P.n_layer) prefetch_phase(P.layers[li + 1].w_qkv, 3 * D, D);
        grid_sync(P.sync, target, sh);
    }
    // final LN + tied-embedding logits
    gemv_phase<RB, true>(P.emb, P.cfg.n_vocab, D, D, nullptr, P.x, D, P.ln_g, P.ln_b, P.logits, P.cfg.n_vocab, EPI_STORE, sh, xs);
    grid_sync(P.sync, target, sh);
}

__device__ __noinline__ void select_phase(const WtsDecodeSteps& P, MgShared& sh)
{
    for (int i = blockIdx.x; i < sh.n_active; i += gridDim.x) {
        const int row = sh.list[i];
        select_row<true>(P.logits + (int64_t)row * P.cfg.n_vocab, P.cfg, P.suppress, P.blank,
                         P.tokens + (int64_t)row * P.cfg.tokens_ld, P.n_tokens + row, __ldg(P.n_prompt + row), P.done + row,
                         P.logprobs + (int64_t)row * P.lp_ld,
                         P.full != nullptr ? P.full + (int64_t)row * P.lp_ld * P.cfg.n_vocab : nullptr,
                         P.last_full != nullptr ? P.last_full + (int64_t)row * P.cfg.n_vocab : nullptr, sh.sel);
        __syncthreads();
    }
}

// RB = activation rows per weight pass (4, 8 or 16): chosen by the host from the number of active rows at launch
// (it only shrinks during a launch); more rows than RB simply take several passes.
template <int RB>
__global__ void __launch_bounds__(MG_THREADS, 1)
decode_steps_kernel(const WtsDecodeSteps P, const int kv_pf_rows)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MgShared& sh = *reinterpret_cast<MgShared*>(smem_raw);
    float* xs = reinterpret_cast<float*>(smem_raw + 1024);    // [MG_MAXROWS][D] staging (aliased by the attention scratch)
    static_assert(sizeof(MgShared) <= 1024, "MgShared must fit its slot");
    uint32_t target = 0;
    if (threadIdx.x == 0) {
        sh.abort_flag = 0;
        sh.prof = blockIdx.x == 0 ? reinterpret_cast<unsigned long long*>(P.prof) : nullptr;
        sh.prof_cap = P.prof_cap;
        sh.prof_idx = 0;
        if (sh.prof != nullptr && sh.prof_cap > 0) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            sh.prof[sh.prof_idx++] = t;
        }
    }
    const int D = P.D;

    for (int step = 0; step < P.n_steps; ++step) {
        // ---- active rows (every CTA builds the same list; `done` was settled before the last barrier)
        __syncthreads();
        if (threadIdx.x < 32) {
            int count = 0;
            for (int b0 = 0; b0 < P.cap; b0 += 32) {
                const int b = b0 + threadIdx.x;
                const bool act = b < P.cap && __ldcg(P.done + b) == 0;
                const unsigned bal = __ballot_sync(FULL_MASK, act);
                const int at = count + __popc(bal & ((1u << threadIdx.x) - 1u));
                if (act && at < MG_MAXROWS) sh.list[at] = b;
                count += __popc(bal);
            }
            if (threadIdx.x == 0) sh.n_active = count;
        }
        __syncthreads();
        const int nA = sh.n_active;
        if (nA == 0 || nA > MG_MAXROWS || sh.abort_flag) break;         // uniform over the grid

        // ---- embed: x[row] = token_embedding[last token] + positional_embedding[its position]
        for (int i = blockIdx.x; i < nA; i += gridDim.x) {
            const int row = sh.list[i];
            const int nt = __ldcg(P.n_tokens + row);
            const int tok = __ldcg(P.tokens + (int64_t)row * P.cfg.tokens_ld + nt - 1);
            const float* e = P.emb + (int64_t)tok * D;
            const float* p = P.pos + (int64_t)(nt - 1) * D;
            for (int c = threadIdx.x; c < D; c += MG_THREADS) P.x[(int64_t)row * D + c] = __ldg(e + c) + __ldg(p + c);
        }
        if (step == 0) prefetch_phase(P.layers[0].w_qkv, 3 * D, D);
        grid_sync(P.sync, target, sh);

        decode_layers_and_logits<RB>(P, sh, xs, target, kv_pf_rows);

        // ---- filters + log-softmax + greedy choice: one CTA per active row
        select_phase(P, sh);
        if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(P.sync + 2, 1u);   // steps completed
        grid_sync(P.sync, target, sh);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// The same step as a chain of LEAN kernels (one per phase), launched with programmatic dependent launch and replayed
// as one CUDA graph.  A software grid barrier costs microseconds (atomics + polling through L2), and the persistent
// kernel needs 259 of them per step even for one active window (tools/step_probe.py times both variants).  A kernel
// boundary under PDL is cheaper, and the next kernel's independent prologue
// (pulling its weight rows into L2) runs while the previous one drains.  Same device code per phase.
__device__ __forceinline__ void build_row_list(const WtsDecodeSteps& P, MgShared& sh)
{
    if (threadIdx.x < 32) {
        int count = 0;
        for (int b0 = 0; b0 < P.cap; b0 += 32) {
            const int b = b0 + threadIdx.x;
            const bool act = b < P.cap && __ldcg(P.done + b) == 0;
            const unsigned bal = __ballot_sync(FULL_MASK, act);
            const int at = count + __popc(bal & ((1u << threadIdx.x) - 1u));
            if (act && at < MG_MAXROWS) sh.list[at] = b;
            count += __popc(bal);
        }
        if (threadIdx.x == 0) { sh.n_active = count <= MG_MAXROWS ? count : 0; sh.abort_flag = 0; sh.prof = nullptr; }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(MG_THREADS)
lean_embed_kernel(const WtsDecodeSteps P)
{
    pdl_launch();
    pdl_wait();
    const int row = blockIdx.x;
    if (row >= P.cap || __ldcg(P.done + row) != 0) return;
    const int nt = __ldcg(P.n_tokens + row);
    const int tok = __ldcg(P.tokens + (int64_t)row * P.cfg.tokens_ld + nt - 1);
    const float* e = P.emb + (int64_t)tok * P.D;
    const float* p = P.pos + (int64_t)(nt - 1) * P.D;
    for (int c = threadIdx.x; c < P.D; c += MG_THREADS) P.x[(int64_t)row * P.D + c] = __ldg(e + c) + __ldg(p + c);
}

template <int RB, bool LN>
__global__ void __launch_bounds__(MG_THREADS, 1)
lean_gemv_kernel(const WtsDecodeSteps P, const float* __restrict__ W, int N, int K, const float* __restrict__ bias,
                 const float* src, int64_t lds, const float* gam, const float* bet, float* out, int64_t ldo, int epi)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MgShared& sh = *reinterpret_cast<MgShared*>(smem_raw);
    float* xs = reinterpret_cast<float*>(smem_raw + 1024);
    pdl_launch();
    prefetch_phase(W, N, K, 3);                              // this CTA's first weight rows -> L2 while the producer drains
    pdl_wait();
    build_row_list(P, sh);
    if (sh.n_active == 0) return;
    gemv_phase<RB, LN>(W, N, K, P.D, bias, src, lds, gam, bet, out, ldo, epi, sh, xs);
}

__global__ void __launch_bounds__(MG_THREADS)
lean_self_attn_kernel(const WtsDecodeSteps P, const WtsDecLayer* Lr)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MgShared& sh = *reinterpret_cast<MgShared*>(smem_raw);
    float* xs = reinterpret_cast<float*>(smem_raw + 1024);
    pdl_launch();
    pdl_wait();
    build_row_list(P, sh);
    const int warp = threadIdx.x >> 5;
    const int t = blockIdx.x * MG_WARPS + warp;
    if (t >= sh.n_active * P.H) return;
    const int row = sh.list[t / P.H];
    self_attention_task(P, *Lr, row, t % P.H, __ldcg(P.n_tokens + row) - 1, xs + warp * P.n_ctx);
}

__global__ void __launch_bounds__(MG_THREADS)
lean_cross_attn_kernel(const WtsDecodeSteps P, const WtsDecLayer* Lr)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MgShared& sh = *reinterpret_cast<MgShared*>(smem_raw);
    float* xs = reinterpret_cast<float*>(smem_raw + 1024);
    pdl_launch();
    pdl_wait();
    build_row_list(P, sh);
    if (blockIdx.x >= sh.n_active * P.H) return;
    cross_attention_phase(P, *Lr, sh, xs);
}

constexpr int LEAN_SELECT_THREADS = 1024;    // one CTA per row walks 51866 logits: 4x the threads of the other lean kernels
__global__ void __launch_bounds__(LEAN_SELECT_THREADS)
lean_select_kernel(const WtsDecodeSteps P)
{
    __shared__ SelectScratch S;
    pdl_launch();
    pdl_wait();
    const int row = blockIdx.x;
    if (row >= P.cap || P.done[row] != 0) return;
    select_row<false>(P.logits + (int64_t)row * P.cfg.n_vocab, P.cfg, P.suppress, P.blank, P.tokens + (int64_t)row * P.cfg.tokens_ld,
                      P.n_tokens + row, P.n_prompt[row], P.done + row, P.logprobs + (int64_t)row * P.lp_ld,
                      P.full != nullptr ? P.full + (int64_t)row * P.lp_ld * P.cfg.n_vocab : nullptr,
                      P.last_full != nullptr ? P.last_full + (int64_t)row * P.cfg.n_vocab : nullptr, S);
}

// ------------------------------------------------------------------------------------------------------------------
// Tensor-core variant of the lean matrix-vector phase: mma.sync.m16n8k16 (bf16 in, float32 accumulate) with the same
// 3-term split-bf16 product as the wgmma GEMMs (hi*hi + lo*hi + hi*lo), but none of their per-kernel set-up (no
// mbarrier ring, no tensor maps, no cluster): at 5..32 active windows the FP32-pipe version above is bound by shared-memory
// loads (an LDS.128 per 16 FMAs), this one by the weight stream.
//  * a CTA owns 8 output features per task; its 8 warps split K; each lane's weight fragment for TWO MMAs is ONE 16-byte
//    load (8 consecutive k of feature n0 + lane/4, both SB16 planes) — made possible by a PERMUTED k order inside every
//    32-k block: activations are staged as bf16x2 words with word 4 s + q <- k = 8 q + 2 s + {0, 1} (tests/dtw_kernel_model.py
//    mma_model checks the algebra), so the A fragments are plain 32-bit shared-memory loads (row pitch K + 8 bf16: conflict-free);
//  * partial 16 x 8 tiles of the 8 warps are summed in shared memory in a fixed order; rows = active windows (16 per m-tile).
__device__ __forceinline__ void mma_m16n8k16_bf16(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                                  uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint4 ldg_stream_u4(const void* p)
{
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo_k, float hi_k)      // lower 16 bits = lower k index
{
    const __nv_bfloat162 v = __floats2bfloat162_rn(lo_k, hi_k);
    return *reinterpret_cast<const uint32_t*>(&v);
}

constexpr int MM_TASK_N = 8;

// staging of one K chunk (kc columns from col0) of the active rows as permuted split-bf16 words; LayerNorm optional
template <bool LN>
__device__ __forceinline__ void mma_stage(const float* src, int64_t ld, int col0, int kc, const float* __restrict__ gam,
                                          const float* __restrict__ bet, const MgShared& sh, uint32_t* Ah, uint32_t* Al, int pitchW)
{
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int NI = kc >> 7;
    for (int i = warp; i < sh.n_active; i += MG_WARPS) {
        const float* r = src + (int64_t)sh.list[i] * ld + col0;
        float4 v[MG_MAXNI];
#pragma unroll
        for (int k = 0; k < MG_MAXNI; ++k)
            if (k < NI) v[k] = ldcg4(r + 4 * (lane + 32 * k));
        if (LN) {
            float s = 0.f;
#pragma unroll
            for (int k = 0; k < MG_MAXNI; ++k)
                if (k < NI) s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
            const float mean = warp_sum(s) / (float)kc;
            float q = 0.f;
#pragma unroll
            for (int k = 0; k < MG_MAXNI; ++k)
                if (k < NI) {
                    const float a = v[k].x - mean, b = v[k].y - mean, c = v[k].z - mean, d = v[k].w - mean;
                    q += (a * a + b * b) + (c * c + d * d);
                }
            const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)kc + 1e-5f);
#pragma unroll
            for (int k = 0; k < MG_MAXNI; ++k)
                if (k < NI) {
                    const float4 g = __ldg(reinterpret_cast<const float4*>(gam) + lane + 32 * k);
                    const float4 b = __ldg(reinterpret_cast<const float4*>(bet) + lane + 32 * k);
                    v[k].x = (v[k].x - mean) * rstd * g.x + b.x;
                    v[k].y = (v[k].y - mean) * rstd * g.y + b.y;
                    v[k].z = (v[k].z - mean) * rstd * g.z + b.z;
                    v[k].w = (v[k].w - mean) * rstd * g.w + b.w;
                }
        }
#pragma unroll
        for (int k = 0; k < MG_MAXNI; ++k)
            if (k < NI) {
                const int f = lane + 32 * k;                 // float4 index: actual k = 4 f .. 4 f + 3
                const int kb = f >> 3, j = f & 7;
                const int w0 = kb * 16 + ((j & 1) * 2) * 4 + (j >> 1);     // word of (k, k+1): s = 2 (j & 1), q = j >> 1
                const float hx = __bfloat162float(__float2bfloat16_rn(v[k].x)), hy = __bfloat162float(__float2bfloat16_rn(v[k].y));
                const float hz = __bfloat162float(__float2bfloat16_rn(v[k].z)), hw = __bfloat162float(__float2bfloat16_rn(v[k].w));
                uint32_t* ah = Ah + (int64_t)i * pitchW;
                uint32_t* al = Al + (int64_t)i * pitchW;
                ah[w0] = pack_bf16x2(hx, hy);
                ah[w0 + 4] = pack_bf16x2(hz, hw);            // (k+2, k+3): s + 1
                al[w0] = pack_bf16x2(v[k].x - hx, v[k].y - hy);
                al[w0 + 4] = pack_bf16x2(v[k].z - hz, v[k].w - hw);
            }
    }
}

template <int MT>
__global__ void __launch_bounds__(MG_THREADS, 1)
lean_mma_kernel(const WtsDecodeSteps P, const __nv_bfloat16* __restrict__ Whi, int64_t plane, int N, int K,
                const float* __restrict__ bias, const float* src, int64_t lds, const float* gam, const float* bet, float* out,
                int64_t ldo, int epi, int ln)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    MgShared& sh = *reinterpret_cast<MgShared*>(smem_raw);
    const int D = P.D;
    const int KC = D;                                        // K is D or 4 D: chunks of D columns
    const int nchunks = K / KC;
    const int pitchW = (KC + 8) >> 1;                        // words per staged row (+8 bf16: rows shift by 16 bytes -> no bank conflicts)
    uint32_t* Ah = reinterpret_cast<uint32_t*>(smem_raw + 1024);
    uint32_t* Al = Ah + (size_t)16 * MT * pitchW;
    float4* red = reinterpret_cast<float4*>(Al + (size_t)16 * MT * pitchW);   // [8 warps][MT][32 lanes]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, q = lane & 3;
    const int ntasks = (N + MM_TASK_N - 1) / MM_TASK_N;
    pdl_launch();
    {   // this CTA's first weight rows -> L2 while the producer drains (both planes)
        const int lines_per_row = K / 64;                    // 128-byte lines of bf16
        for (int t = blockIdx.x, r = 0; t < ntasks && r < 2; t += gridDim.x, ++r)
            for (int ln_ = threadIdx.x; ln_ < MM_TASK_N * lines_per_row * 2; ln_ += MG_THREADS) {
                const int pl = ln_ / (MM_TASK_N * lines_per_row), rem = ln_ - pl * MM_TASK_N * lines_per_row;
                const int f = rem / lines_per_row, c = rem - f * lines_per_row;
                prefetch_l2(Whi + (int64_t)pl * plane + (int64_t)min(t * MM_TASK_N + f, N - 1) * K + c * 64);
            }
    }
    pdl_wait();
    build_row_list(P, sh);
    const int nA = sh.n_active;
    if (nA == 0) return;
    // rows of the m-tiles beyond the active ones stay zero (finite), written once
    for (int idx = threadIdx.x; idx < (16 * MT - nA) * pitchW; idx += MG_THREADS) {
        Ah[(size_t)nA * pitchW + idx] = 0u;
        Al[(size_t)nA * pitchW + idx] = 0u;
    }
    const int nkb = KC >> 5;
    float acc[2][MT][4];                                     // K in several chunks (FC2): at most 2 tasks per CTA, kept across chunks
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[r][m][e] = 0.f;

    auto task_partial = [&](int t, int c, float (&part)[MT][4]) {
        const int n = min(t * MM_TASK_N + g, N - 1);
        const __nv_bfloat16* wrow = Whi + (int64_t)n * K + (int64_t)c * KC + 8 * q;
#pragma unroll 1
        for (int kb0 = warp; kb0 < nkb; kb0 += 5 * MG_WARPS) {
            uint4 bh[5], bl[5];
#pragma unroll
            for (int u = 0; u < 5; ++u) {
                const int kb = kb0 + u * MG_WARPS;
                if (kb < nkb) {
                    bh[u] = ldg_stream_u4(wrow + kb * 32);
                    bl[u] = ldg_stream_u4(wrow + kb * 32 + plane);
                }
            }
#pragma unroll
            for (int u = 0; u < 5; ++u) {
                const int kb = kb0 + u * MG_WARPS;
                if (kb < nkb) {
#pragma unroll
                    for (int m = 0; m < MT; ++m) {
                        const uint32_t* ah0 = Ah + (size_t)(16 * m + g) * pitchW + kb * 16 + q;
                        const uint32_t* ah8 = ah0 + (size_t)8 * pitchW;
                        const uint32_t* al0 = Al + (size_t)(16 * m + g) * pitchW + kb * 16 + q;
                        const uint32_t* al8 = al0 + (size_t)8 * pitchW;
                        // first MMA of the block: segments S0, S1 with the first two words of the weight load
                        {
                            const uint32_t a0 = ah0[0], a1 = ah8[0], a2 = ah0[4], a3 = ah8[4];
                            const uint32_t l0 = al0[0], l1 = al8[0], l2 = al0[4], l3 = al8[4];
                            mma_m16n8k16_bf16(part[m], a0, a1, a2, a3, bh[u].x, bh[u].y);
                            mma_m16n8k16_bf16(part[m], l0, l1, l2, l3, bh[u].x, bh[u].y);
                            mma_m16n8k16_bf16(part[m], a0, a1, a2, a3, bl[u].x, bl[u].y);
                        }
                        // second MMA: segments S2, S3 with the last two words
                        {
                            const uint32_t a0 = ah0[8], a1 = ah8[8], a2 = ah0[12], a3 = ah8[12];
                            const uint32_t l0 = al0[8], l1 = al8[8], l2 = al0[12], l3 = al8[12];
                            mma_m16n8k16_bf16(part[m], a0, a1, a2, a3, bh[u].z, bh[u].w);
                            mma_m16n8k16_bf16(part[m], l0, l1, l2, l3, bh[u].z, bh[u].w);
                            mma_m16n8k16_bf16(part[m], a0, a1, a2, a3, bl[u].z, bl[u].w);
                        }
                    }
                }
            }
        }
    };
    auto task_finish = [&](int t, float (&part)[MT][4]) {   // fixed-order sum over the 8 warps, epilogue by warps 0 .. MT-1
#pragma unroll
        for (int m = 0; m < MT; ++m) red[(warp * MT + m) * 32 + lane] = make_float4(part[m][0], part[m][1], part[m][2], part[m][3]);
        __syncthreads();
        if (warp < MT) {
            float4 s = red[(0 * MT + warp) * 32 + lane];
#pragma unroll
            for (int w = 1; w < MG_WARPS; ++w) {
                const float4 v = red[(w * MT + warp) * 32 + lane];
                s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
            }
            const float vals[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int ri = 16 * warp + g + ((e >> 1) ? 8 : 0);
                const int n = t * MM_TASK_N + 2 * q + (e & 1);
                if (ri < nA && n < N) {
                    float v = vals[e] + (bias != nullptr ? __ldg(bias + n) : 0.f);
                    float* dst = out + (int64_t)sh.list[ri] * ldo + n;
                    if (epi == EPI_GELU) v = gelu_erf(v);
                    else if (epi == EPI_ADD) v += __ldcg(dst);
                    *dst = v;
                }
            }
        }
        __syncthreads();
    };

    for (int c = 0; c < nchunks; ++c) {
        if (c > 0) __syncthreads();                          // previous chunk fully consumed
        if (ln) mma_stage<true>(src, lds, c * KC, KC, gam, bet, sh, Ah, Al, pitchW);
        else    mma_stage<false>(src, lds, c * KC, KC, nullptr, nullptr, sh, Ah, Al, pitchW);
        __syncthreads();
        if (nchunks == 1) {
            for (int t = blockIdx.x; t < ntasks; t += gridDim.x) {
                float part[MT][4];
#pragma unroll
                for (int m = 0; m < MT; ++m)
#pragma unroll
                    for (int e = 0; e < 4; ++e) part[m][e] = 0.f;
                task_partial(t, 0, part);
                task_finish(t, part);
            }
        } else {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int t = blockIdx.x + r * gridDim.x;
                if (t < ntasks) task_partial(t, c, acc[r]);
            }
        }
    }
    if (nchunks > 1) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int t = blockIdx.x + r * gridDim.x;
            if (t < ntasks) task_finish(t, acc[r]);          // uniform over the CTA
        }
    }
}

template <int MT>
static int launch_lean_step_mma(const WtsDecodeSteps& P, const WtsDecLayer* h_layers, int n_sm, cudaStream_t st)
{
    const int D = P.D, H = P.H, V = P.cfg.n_vocab;
    const int pitchW = (D + 8) >> 1;
    const size_t sm_mma = 1024 + (size_t)2 * 16 * MT * pitchW * 4 + (size_t)MG_WARPS * MT * 32 * 16;
    const size_t sm_self = (size_t)MG_WARPS * P.n_ctx * sizeof(float) + 1024;
    const size_t sm_cross = sizeof(CaScratch) + 1024;
    static bool attr = false;
    if (!attr) {
        WTS_CUDA_CHECK(cudaFuncSetAttribute(lean_mma_kernel<MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
        attr = true;
    }
    if (sm_mma > 200 * 1024) { set_error("wts_decode_step_kernels: %zu bytes of shared memory needed", sm_mma); return -2; }
    const dim3 g_gemv(n_sm), blk(MG_THREADS);
    const dim3 g_self((P.max_rows * H + MG_WARPS - 1) / MG_WARPS), g_cross(P.max_rows * H);
    typedef const __nv_bfloat16* BF;
    const float* nof = nullptr;
    WTS_CUDA_CHECK(launch_pdl(lean_embed_kernel, dim3(P.cap), blk, 0, st, P));
    for (int li = 0; li < P.n_layer; ++li) {
        const WtsDecLayer& L = h_layers[li];
        const WtsDecLayer* dL = P.layers + li;
        WTS_CUDA_CHECK(launch_pdl(lean_mma_kernel<MT>, g_gemv, blk, sm_mma, st, P, (BF)L.sb_qkv, (int64_t)L.pl_qkv, 3 * D, D, L.b_qkv,
                                  (const float*)P.x, (int64_t)D, L.ln1_g, L.ln1_b, P.qkv, (int64_t)(3 * D), (int)EPI_STORE, 1));
        WTS_CUDA_CHECK(launch_pdl(lean_self_attn_kernel, g_self, blk, sm_self, st, P, dL));
        WTS_CUDA_CHECK(launch_pdl(lean_mma_kernel<MT>, g_gemv, blk, sm_mma, st, P, (BF)L.sb_o, (int64_t)L.pl_o, D, D, L.b_o,
                                  (const float*)P.att, (int64_t)D, nof, nof, P.x, (int64_t)D, (int)EPI_ADD, 0));
        WTS_CUDA_CHECK(launch_pdl(lean_mma_kernel<MT>, g_gemv, blk, sm_mma, st, P, (BF)L.sb_cq, (int64_t)L.pl_cq, D, D, L.b_cq,
                                  (const float*)P.x, (int64_t)D, L.ln2_g, L.ln2_b, P.q, (int64_t)D, (int)EPI_STORE, 1));
        WTS_CUDA_CHECK(launch_pdl(lean_cross_attn_kernel, g_cross, blk, sm_cross, st, P, dL));
        WTS_CUDA_CHECK(launch_pdl(lean_mma_kernel<MT>, g_gemv, blk, sm_mma, st, P, (BF)L.sb_co, (int64_t)L.pl_co, D, D, L.b_co,
                                  (const float*)P.att, (int64_t)D, nof, nof, P.x, (int64_t)D, (int)EPI_ADD, 0));
        WTS_CUDA_CHECK(launch_pdl(lean_mma_kernel<MT>, g_gemv, blk, sm_mma, st, P, (BF)L.sb_fc1, (int64_t)L.pl_fc1, 4 * D, D, L.b_fc1,
                                  (const float*)P.x, (int64_t)D, L.ln3_g, L.ln3_b, P.mid, (int64_t)(4 * D), (int)EPI_GELU, 1));
        WTS_CUDA_CHECK(launch_pdl(lean_mma_kernel<MT>, g_gemv, blk, sm_mma, st, P, (BF)L.sb_fc2, (int64_t)L.pl_fc2, D, 4 * D, L.b_fc2,
                                  (const float*)P.mid, (int64_t)(4 * D), nof, nof, P.x, (int64_t)D, (int)EPI_ADD, 0));
    }
    WTS_CUDA_CHECK(launch_pdl(lean_mma_kernel<MT>, g_gemv, blk, sm_mma, st, P, (BF)P.emb_sb, (int64_t)P.emb_plane, V, D, nof,
                              (const float*)P.x, (int64_t)D, P.ln_g, P.ln_b, P.logits, (int64_t)V, (int)EPI_STORE, 1));
    WTS_CUDA_CHECK(launch_pdl(lean_select_kernel, dim3(P.cap), dim3(LEAN_SELECT_THREADS), 0, st, P));
    return 0;
}

template <int RB>
static int launch_lean_step(const WtsDecodeSteps& P, const WtsDecLayer* h_layers, int n_sm, cudaStream_t st)
{
    const int D = P.D, H = P.H, V = P.cfg.n_vocab;
    const size_t stage = (size_t)MG_STAGE_FLOATS * sizeof(float) + 1024;
    const size_t sm_self = (size_t)MG_WARPS * P.n_ctx * sizeof(float) + 1024;
    const size_t sm_cross = sizeof(CaScratch) + 1024;
    static bool attr = false;
    if (!attr) {
        WTS_CUDA_CHECK(cudaFuncSetAttribute(lean_gemv_kernel<RB, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stage));
        WTS_CUDA_CHECK(cudaFuncSetAttribute(lean_gemv_kernel<RB, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stage));
        attr = true;
    }
    const dim3 g_gemv(n_sm), blk(MG_THREADS);
    const dim3 g_self((P.max_rows * H + MG_WARPS - 1) / MG_WARPS), g_cross(P.max_rows * H);
    WTS_CUDA_CHECK(launch_pdl(lean_embed_kernel, dim3(P.cap), blk, 0, st, P));
    const float* nof = nullptr;
    for (int li = 0; li < P.n_layer; ++li) {
        const WtsDecLayer& L = h_layers[li];
        const WtsDecLayer* dL = P.layers + li;
        WTS_CUDA_CHECK(launch_pdl(lean_gemv_kernel<RB, true>, g_gemv, blk, stage, st, P, L.w_qkv, 3 * D, D, L.b_qkv, (const float*)P.x,
                                  (int64_t)D, L.ln1_g, L.ln1_b, P.qkv, (int64_t)(3 * D), (int)EPI_STORE));
        WTS_CUDA_CHECK(launch_pdl(lean_self_attn_kernel, g_self, blk, sm_self, st, P, dL));
        WTS_CUDA_CHECK(launch_pdl(lean_gemv_kernel<RB, false>, g_gemv, blk, stage, st, P, L.w_o, D, D, L.b_o, (const float*)P.att,
                                  (int64_t)D, nof, nof, P.x, (int64_t)D, (int)EPI_ADD));
        WTS_CUDA_CHECK(launch_pdl(lean_gemv_kernel<RB, true>, g_gemv, blk, stage, st, P, L.w_cq, D, D, L.b_cq, (const float*)P.x,
                                  (int64_t)D, L.ln2_g, L.ln2_b, P.q, (int64_t)D, (int)EPI_STORE));
        WTS_CUDA_CHECK(launch_pdl(lean_cross_attn_kernel, g_cross, blk, sm_cross, st, P, dL));
        WTS_CUDA_CHECK(launch_pdl(lean_gemv_kernel<RB, false>, g_gemv, blk, stage, st, P, L.w_co, D, D, L.b_co, (const float*)P.att,
                                  (int64_t)D, nof, nof, P.x, (int64_t)D, (int)EPI_ADD));
        WTS_CUDA_CHECK(launch_pdl(lean_gemv_kernel<RB, true>, g_gemv, blk, stage, st, P, L.w_fc1, 4 * D, D, L.b_fc1, (const float*)P.x,
                                  (int64_t)D, L.ln3_g, L.ln3_b, P.mid, (int64_t)(4 * D), (int)EPI_GELU));
        WTS_CUDA_CHECK(launch_pdl(lean_gemv_kernel<RB, false>, g_gemv, blk, stage, st, P, L.w_fc2, D, 4 * D, L.b_fc2, (const float*)P.mid,
                                  (int64_t)(4 * D), nof, nof, P.x, (int64_t)D, (int)EPI_ADD));
    }
    WTS_CUDA_CHECK(launch_pdl(lean_gemv_kernel<RB, true>, g_gemv, blk, stage, st, P, P.emb, V, D, nof, (const float*)P.x, (int64_t)D,
                              P.ln_g, P.ln_b, P.logits, (int64_t)V, (int)EPI_STORE));
    WTS_CUDA_CHECK(launch_pdl(lean_select_kernel, dim3(P.cap), dim3(LEAN_SELECT_THREADS), 0, st, P));
    return 0;
}

}  // namespace wts

using namespace wts;

extern "C" int wts_decode_steps(const WtsDecodeSteps* p, void* stream)
{
    if (!p) { set_error("wts_decode_steps: null argument"); return -2; }
    const WtsDecodeSteps& P = *p;
    if (P.D % 128 != 0 || P.D > 128 * MG_MAXNI || P.D != P.H * 64) {
        set_error("wts_decode_steps: n_text_state %d not supported (multiple of 128, <= %d, 64 per head)", P.D, 128 * MG_MAXNI);
        return -2;
    }
    if (P.max_rows > MG_MAXROWS) { set_error("wts_decode_steps: at most %d active rows", MG_MAXROWS); return -2; }
    if (P.n_steps <= 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    static int n_sm = 0, l2_bytes = 0;
    static size_t smem_set = 0;
    if (n_sm == 0) {
        int dev = 0;
        WTS_CUDA_CHECK(cudaGetDevice(&dev));
        WTS_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
        WTS_CUDA_CHECK(cudaDeviceGetAttribute(&l2_bytes, cudaDevAttrL2CacheSize, dev));
    }
    const int64_t kv_row_bytes = 2 * (int64_t)P.H * P.n_audio_ctx * 64 * 2;     // fp16 K + V of one row, one layer
    int kv_pf_rows = (int)((int64_t)l2_bytes / 2 / kv_row_bytes);
    if (kv_pf_rows > MG_KV_PREFETCH_ROWS) kv_pf_rows = MG_KV_PREFETCH_ROWS;
    const size_t stage = (size_t)MG_STAGE_FLOATS * sizeof(float);             // gemv_phase sizes its chunks for this capacity
    size_t smem = stage > sizeof(CaScratch) ? stage : sizeof(CaScratch);
    const size_t sa = (size_t)MG_WARPS * P.n_ctx * sizeof(float);             // self-attention score scratch
    if (sa > smem) smem = sa;
    smem += 1024;
    if (smem > 227 * 1024) { set_error("wts_decode_steps: %zu bytes of shared memory needed", smem); return -2; }
    if (smem > smem_set) {
        WTS_CUDA_CHECK(cudaFuncSetAttribute(decode_steps_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        WTS_CUDA_CHECK(cudaFuncSetAttribute(decode_steps_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        WTS_CUDA_CHECK(cudaFuncSetAttribute(decode_steps_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        smem_set = smem;
    }
    WTS_CUDA_CHECK(cudaMemsetAsync(P.sync, 0, 64 * sizeof(uint32_t), st));
    void* args[] = {const_cast<WtsDecodeSteps*>(p), &kv_pf_rows};
    const void* fn = P.max_rows <= 4 ? (const void*)decode_steps_kernel<4>
                   : P.max_rows <= 8 ? (const void*)decode_steps_kernel<8> : (const void*)decode_steps_kernel<16>;
    WTS_CUDA_CHECK(cudaLaunchCooperativeKernel(fn, dim3(n_sm), dim3(MG_THREADS), args, smem, st));
    return 0;
}

static bool D_ok_for_mma(const WtsDecodeSteps& P)
{
    // K chunks of D columns, 32-k blocks, at most two 8-feature tasks per CTA for the 4D-wide FC2, SB16 planes present
    return P.D % 128 == 0 && P.emb_sb != nullptr && (P.D / MM_TASK_N) <= 2 * 132;
}

// One decoder step as a chain of per-phase kernels (same arithmetic as wts_decode_steps; see the comment above
// lean_embed_kernel).  h_layers: HOST copy of the layer table (weight pointers become kernel arguments).  Capturable in a
// CUDA graph: no host synchronisation, no memset.  2 + 8 n_layer + 1 launches.
extern "C" int wts_decode_step_kernels(const WtsDecodeSteps* p, const WtsDecLayer* h_layers, void* stream)
{
    if (!p || !h_layers) { set_error("wts_decode_step_kernels: null argument"); return -2; }
    const WtsDecodeSteps& P = *p;
    if (P.D % 128 != 0 || P.D > 128 * MG_MAXNI || P.D != P.H * 64) {
        set_error("wts_decode_step_kernels: n_text_state %d not supported", P.D);
        return -2;
    }
    if (P.max_rows > MG_MAXROWS || P.max_rows < 1) { set_error("wts_decode_step_kernels: 1..%d active rows", MG_MAXROWS); return -2; }
    if ((size_t)MG_WARPS * P.n_ctx * sizeof(float) + 1024 > 48 * 1024) { set_error("wts_decode_step_kernels: n_text_ctx too large"); return -2; }
    static int n_sm = 0;
    if (n_sm == 0) {
        int dev = 0;
        WTS_CUDA_CHECK(cudaGetDevice(&dev));
        WTS_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (P.use_mma) {
        if (D_ok_for_mma(P)) return P.max_rows <= 16 ? launch_lean_step_mma<1>(P, h_layers, n_sm, st)
                                                     : launch_lean_step_mma<2>(P, h_layers, n_sm, st);
    }
    if (P.max_rows <= 4) return launch_lean_step<4>(P, h_layers, n_sm, st);
    if (P.max_rows <= 8) return launch_lean_step<8>(P, h_layers, n_sm, st);
    return launch_lean_step<16>(P, h_layers, n_sm, st);
}
