// Decoder step for SMALL active batches (<= 32 windows still decoding) as a chain of lean per-phase kernels.
//
// Why: a decoder step of large-v3 is ~355 dependent kernels when every operator is its own launch; at a few active
// windows each of them sits at its launch + prologue floor, far above the time the step's weight stream needs from HBM.
// Here one step is 2 + 8 n_layer + 1 kernels,
//     embed -> L x [LN+QKV | self-attn | out-proj | LN+Q | cross-attn | out-proj | LN+FC1+GELU | FC2] -> LN+logits -> select
// launched with programmatic dependent launch and replayed as one CUDA graph: a kernel boundary under PDL is cheap,
// and each matrix-vector kernel pulls its first weight rows into L2 while the previous kernel drains.  Cross-attention
// K/V are streamed by the cross-attention kernel itself; nothing prefetches them.
// Replaces, for the whole batch at once, upstream's DecodingTask._main_loop step + the reference's per-token hooks
// (T.py:783-793 hook_attention_weights, 849-881 hook_output_logits).
//
// The matrix-vector phases run on mma.sync tensor cores with the SB16 weight planes (see lean_mma_kernel); attention,
// LayerNorm statistics, the filters and the choice stay in float32.  The kernels find the active rows from the done
// flags on the device, so one graph serves every step; only the grid sizes depend on the host's bound `max_rows`.
#include "decode_common.cuh"

namespace wts {

constexpr int MG_THREADS = 256;
constexpr int MG_WARPS = MG_THREADS / 32;
constexpr int MG_MAXROWS = 32;          // active rows a step handles
constexpr int MG_MAXNI = 10;            // D / 128 <= 10 (D <= 1280)

struct MgShared {
    int list[MG_MAXROWS];               // active slots, ascending
    int n_active;
};

__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

enum { EPI_STORE = 0, EPI_ADD = 1, EPI_GELU = 2 };

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
            kal = Lr.cross_k_align + ((int64_t)row * Lr.align_n + slot - Lr.align_s0) * P.n_audio_ctx * 64;
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
        if (threadIdx.x == 0) sh.n_active = count <= MG_MAXROWS ? count : 0;
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
    select_row(P.logits + (int64_t)row * P.cfg.n_vocab, P.cfg, P.suppress, P.blank, P.tokens + (int64_t)row * P.cfg.tokens_ld,
               P.n_tokens + row, P.n_prompt[row], P.done + row, P.logprobs + (int64_t)row * P.lp_ld,
               P.full != nullptr ? P.full + (int64_t)row * P.lp_ld * P.cfg.n_vocab : nullptr,
               P.last_full != nullptr ? P.last_full + (int64_t)row * P.cfg.n_vocab : nullptr, S);
}

// ------------------------------------------------------------------------------------------------------------------
// The lean matrix-vector phase: mma.sync.m16n8k16 (bf16 in, float32 accumulate) with the same 3-term split-bf16
// product as the wgmma GEMMs (hi*hi + lo*hi + hi*lo), but none of their per-kernel set-up (no mbarrier ring, no tensor
// maps, no cluster), so at a few active windows it is bound by the weight stream.
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
static int launch_lean_step(const WtsDecodeSteps& P, const WtsDecLayer* h_layers, int n_sm, cudaStream_t st)
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

}  // namespace wts

using namespace wts;

// One decoder step as a chain of per-phase kernels (see the comment at the top).  h_layers: HOST copy of the layer
// table (weight pointers become kernel arguments).  Capturable in a CUDA graph: no host synchronisation, no memset.
// 2 + 8 n_layer + 1 launches.
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
    if (P.emb_sb == nullptr) { set_error("wts_decode_step_kernels: no SB16 token embedding"); return -2; }
    static int n_sm = 0;
    if (n_sm == 0) {
        int dev = 0;
        WTS_CUDA_CHECK(cudaGetDevice(&dev));
        WTS_CUDA_CHECK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    }
    // lean_mma_kernel's grid is one CTA per SM, and with K = 4 D (FC2) a CTA keeps at most two 8-feature tasks
    // across the K chunks: fewer than D / 16 SMs would leave FC2 outputs uncomputed
    if (P.D / MM_TASK_N > 2 * n_sm) {
        set_error("wts_decode_step_kernels: n_text_state %d needs at least %d SMs, the device has %d", P.D, P.D / 16, n_sm);
        return -2;
    }
    cudaStream_t st = (cudaStream_t)stream;
    return P.max_rows <= 16 ? launch_lean_step<1>(P, h_layers, n_sm, st) : launch_lean_step<2>(P, h_layers, n_sm, st);
}
