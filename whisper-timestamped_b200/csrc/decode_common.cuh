// Device code shared by the per-kernel decode step (ops.cu) and the lean small-batch decode step
// (decode_steps.cu): block reductions, the one-pass fp16 cross-attention stream, and the fused
// logit-filter / log-softmax / greedy-argmax of one sequence.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math_constants.h>

#include "common.cuh"

namespace wts {

__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo)
{
    hi = __float2bfloat16_rn(x);
    lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

__device__ __forceinline__ float block_reduce_sum(float v, float* red)
{
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (l == 0) red[w] = v;
    __syncthreads();
    float r = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
    if (w == 0) { r = warp_sum(r); if (l == 0) red[0] = r; }
    __syncthreads();
    return red[0];
}
__device__ __forceinline__ float block_reduce_max(float v, float* red)
{
    v = warp_max(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (l == 0) red[w] = v;
    __syncthreads();
    float r = (threadIdx.x < nw) ? red[threadIdx.x] : -CUDART_INF_F;
    if (w == 0) { r = warp_max(r); if (l == 0) red[0] = r; }
    __syncthreads();
    return red[0];
}

__device__ __forceinline__ float gelu_erf(float v) { return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f)); }

// -------------------------------------------------------------- cross attention, fp16 K/V caches
// A CTA of CA_THREADS = 32 key groups x 8 lanes; a lane owns 8 of the 64 channels.  Group g streams keys g, g+32, ...:
// K row (16 B/lane fp16, or 32 B/lane from the float32 alignment copy) and V row (16 B/lane) are loaded UNROLL keys
// ahead (coalesced 128-byte rows), the score is an 8-lane shuffle reduction and softmax x V is accumulated ONLINE
// (running max / sum), so K and V are streamed exactly once with no score buffer.  Raw scores of the alignment heads
// go to qk_dst on the way (T.py:783-793: the reference's "attention weights" are these pre-softmax rows).
constexpr int CA_THREADS = 256;
constexpr int CA_GROUPS = CA_THREADS / 8;

template <bool KF32, int UNROLL>
__device__ __forceinline__ void ca_stream(const void* __restrict__ Kbase, const __half* __restrict__ Vbase, int ctx, int g,
                                          int c8, const float (&qf)[8], float* __restrict__ qk_dst, float& m, float& l,
                                          float (&acc)[8])
{
    for (int j0 = g; j0 < ctx; j0 += CA_GROUPS * UNROLL) {
        uint4 kr[UNROLL][KF32 ? 2 : 1];
        uint4 vr[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const int j = min(j0 + CA_GROUPS * u, ctx - 1);
            if (KF32) {
                const uint4* p = reinterpret_cast<const uint4*>(static_cast<const float*>(Kbase) + (int64_t)j * 64 + c8 * 8);
                kr[u][0] = __ldcs(p);
                kr[u][KF32 ? 1 : 0] = __ldcs(p + 1);
            } else {
                kr[u][0] = __ldcs(reinterpret_cast<const uint4*>(static_cast<const __half*>(Kbase) + (int64_t)j * 64 + c8 * 8));
            }
            vr[u] = __ldcs(reinterpret_cast<const uint4*>(Vbase + (int64_t)j * 64 + c8 * 8));
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const int j = j0 + CA_GROUPS * u;
            const bool valid = j < ctx;
            float s = 0.f;
            if (KF32) {
                const float* kf = reinterpret_cast<const float*>(&kr[u][0]);
#pragma unroll
                for (int e = 0; e < 8; ++e) s += qf[e] * kf[e];
            } else {
                const __half2* h2 = reinterpret_cast<const __half2*>(&kr[u][0]);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 f = __half22float2(h2[e]);
                    s += qf[2 * e] * f.x + qf[2 * e + 1] * f.y;
                }
            }
            s += __shfl_xor_sync(0xffffffffu, s, 1);
            s += __shfl_xor_sync(0xffffffffu, s, 2);
            s += __shfl_xor_sync(0xffffffffu, s, 4);
            if (valid && qk_dst != nullptr && c8 == 0) qk_dst[j] = s;
            const float mn = fmaxf(m, valid ? s : -1e30f);
            const float sc = __expf(m - mn);
            const float p = valid ? __expf(s - mn) : 0.f;
            l = l * sc + p;
            const __half2* v2 = reinterpret_cast<const __half2*>(&vr[u]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = __half22float2(v2[e]);
                acc[2 * e] = acc[2 * e] * sc + p * f.x;
                acc[2 * e + 1] = acc[2 * e + 1] * sc + p * f.y;
            }
            m = mn;
        }
    }
}

// Shared-memory scratch of one (query row, head) cross-attention: the 32 partial (max, sum, acc) triples.
struct CaScratch {
    float acc[CA_GROUPS][64];
    float m[CA_GROUPS], l[CA_GROUPS], w[CA_GROUPS];
    float L;
};

// One (query row, head) by a CTA of CA_THREADS threads.  qf: this lane's 8 query channels.  Returns (threads < 64)
// the output channel threadIdx.x in `y`; all threads must call it (it synchronises the CTA).
template <int UNROLL>
__device__ __forceinline__ float ca_row_head(const float (&qf)[8], const __half* k16, const __half* v16, const float* k_align,
                                             float* qk_dst, int ctx, CaScratch& sc)
{
    const int c8 = threadIdx.x & 7, g = threadIdx.x >> 3;
    float m = -1e30f, l = 0.f;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (k_align != nullptr) ca_stream<true, UNROLL>(k_align, v16, ctx, g, c8, qf, qk_dst, m, l, acc);
    else                    ca_stream<false, UNROLL>(k16, v16, ctx, g, c8, qf, nullptr, m, l, acc);
    if (c8 == 0) { sc.m[g] = m; sc.l[g] = l; }
    *reinterpret_cast<float4*>(&sc.acc[g][c8 * 8]) = make_float4(acc[0], acc[1], acc[2], acc[3]);
    *reinterpret_cast<float4*>(&sc.acc[g][c8 * 8 + 4]) = make_float4(acc[4], acc[5], acc[6], acc[7]);
    __syncthreads();
    if (threadIdx.x < 32) {
        const float mg = sc.m[threadIdx.x];
        const float M = warp_max(mg);
        const float w = __expf(mg - M);
        sc.w[threadIdx.x] = w;
        const float L = warp_sum(sc.l[threadIdx.x] * w);
        if (threadIdx.x == 0) sc.L = L;
    }
    __syncthreads();
    float y = 0.f;
    if (threadIdx.x < 64) {
#pragma unroll
        for (int gg = 0; gg < CA_GROUPS; ++gg) y += sc.acc[gg][threadIdx.x] * sc.w[gg];
        y /= sc.L;
    }
    return y;
}

// ------------------------------------------------------------------------------------ decode select
// Logit filters + log-softmax + greedy choice of ONE sequence by the whole CTA (any block size that is a multiple of
// 32, <= 1024) — replaces SuppressBlank / SuppressTokens / ApplyTimestampRules / GreedyDecoder.update (upstream
// whisper.decoding; rebuilt by the reference at T.py:1371-1393 and re-applied in hook_output_logits, T.py:871-875).
// `last_full`: when this step reaches the decoding limit the whole filtered log-softmax row is
// kept (one row per sequence) — the reference reads chunk_logprobs[-1][fallback_token] there (T.py:529-538, 735).
struct SelectScratch {
    float red[32];
    int flags[8];
    float best[32];
    int besti[32];
};

__device__ __forceinline__ void select_row(const float* x, const WtsDecodeCfg& cfg, const uint8_t* __restrict__ suppress,
                                           const uint8_t* __restrict__ blank, int32_t* tk, int32_t* n_tokens_b, int np,
                                           int32_t* done_b, float* logprobs_b, float* full_b, float* last_full_b,
                                           SelectScratch& S, const bool rows_only = false)
{
    // rows_only: only write the filtered log-softmax row to full_b[0 .. V) — no choice, no state update (what beam
    // search / sampling consume: upstream BeamSearchDecoder.update / GreedyDecoder.update work on these rows)
    const int T = blockDim.x;
    const int nt = *n_tokens_b;
    const int n = nt - np;                                   // sampled so far
    const int V = cfg.n_vocab, tsb = cfg.timestamp_begin, eot = cfg.eot;
    // ---- token history: position of the last sampled timestamp (parallel scan, no dependent chain)
    int last_pos = -1;
    for (int i = np + threadIdx.x; i < nt; i += T)
        if (tk[i] >= tsb) last_pos = i;                      // ascending i per thread
    last_pos = (int)block_reduce_max((float)last_pos, S.red);   // positions < 2^24: exact in float
    if (threadIdx.x == 0) {
        const bool last_ts = n >= 1 && tk[nt - 1] >= tsb;
        const bool pen_ts = n < 2 || tk[nt - 2] >= tsb;
        const int tl = last_pos >= 0 ? tk[last_pos] : -1;
        int ts_limit = tsb;                                  // timestamps in [tsb, ts_limit) are forbidden
        if (tl >= 0) ts_limit = (last_ts && !pen_ts) ? tl : tl + 1;
        S.flags[0] = (n == 0);
        S.flags[1] = last_ts && pen_ts;                      // forbid all timestamps
        S.flags[2] = last_ts && !pen_ts;                     // forbid text below eot
        S.flags[3] = ts_limit;
    }
    __syncthreads();
    const bool first = S.flags[0], no_ts = S.flags[1], no_text = S.flags[2];
    const int ts_limit = S.flags[3];
    const int ts_max = (first && cfg.max_initial_ts >= 0) ? tsb + cfg.max_initial_ts : V;

    // rules that only depend on the index (the per-token masks are loaded alongside the logits)
    auto range_ok = [&](int v) -> bool {
        if (v == cfg.no_timestamps) return false;
        if (v >= tsb) return !(no_ts || v < ts_limit || v > ts_max);
        return !(first || (no_text && v < eot));
    };

    // ---- ONE pass over the row, 8 independent loads in flight per thread: running (max, sum of exp, argmax) of the
    // allowed text tokens and of the allowed timestamp tokens
    constexpr int UN = 8;
    float mt = -CUDART_INF_F, st = 0.f, ms = -CUDART_INF_F, ss = 0.f;
    int bti = 0x7fffffff, bsi = 0x7fffffff;                  // argmax of each set (value = mt / ms)
    for (int v0 = threadIdx.x; v0 < V; v0 += UN * T) {
        float xv[UN];
        unsigned bad = 0;
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const int v = v0 + u * T;
            const bool in = v < V;
            xv[u] = in ? x[v] : 0.f;
            const unsigned b = in ? (unsigned)__ldg(suppress + v) | (first ? (unsigned)__ldg(blank + v) : 0u) : 1u;
            bad |= (b != 0u ? 1u : 0u) << u;
        }
#pragma unroll
        for (int u = 0; u < UN; ++u) {
            const int v = v0 + u * T;
            if (((bad >> u) & 1u) || !range_ok(v)) continue;
            const float xx = xv[u];
            if (v >= tsb) {                                  // ascending v per thread: the first maximum is kept
                if (xx > ms) { ss = ss * expf(ms - xx) + 1.f; ms = xx; bsi = v; } else ss += expf(xx - ms);
            } else {
                if (xx > mt) { st = st * expf(mt - xx) + 1.f; mt = xx; bti = v; } else st += expf(xx - mt);
            }
        }
    }
    const float Mt = block_reduce_max(mt, S.red);
    const float Ms = block_reduce_max(ms, S.red);
    const float St = block_reduce_sum(mt > -CUDART_INF_F ? st * expf(mt - Mt) : 0.f, S.red);
    const float Ss = block_reduce_sum(ms > -CUDART_INF_F ? ss * expf(ms - Ms) : 0.f, S.red);
    const float lse_ts = (Ms > -CUDART_INF_F) ? Ms + logf(Ss) : -CUDART_INF_F;
    const bool only_ts = lse_ts > Mt;                        // "sum of timestamp probability beats any text token"
    // block argmax over the final allowed set, lowest index on ties
    {
        const bool take_text = !only_ts && mt >= ms;         // equal values: the lower index (a text token) wins
        float bv = take_text ? mt : ms;
        int bi = take_text ? bti : bsi;
        if (bv == -CUDART_INF_F) bi = 0x7fffffff;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(FULL_MASK, bv, o);
            const int oi = __shfl_xor_sync(FULL_MASK, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if ((threadIdx.x & 31) == 0) { S.best[threadIdx.x >> 5] = bv; S.besti[threadIdx.x >> 5] = bi; }
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < T / 32; ++w)
                if (S.best[w] > bv || (S.best[w] == bv && S.besti[w] < bi)) { bv = S.best[w]; bi = S.besti[w]; }
            S.best[0] = bv; S.besti[0] = bi;
        }
        __syncthreads();
    }
    float lse;
    if (only_ts) {
        lse = lse_ts;
    } else {
        const float gm = fmaxf(Mt, Ms);
        const float sum = (Mt > -CUDART_INF_F ? St * expf(Mt - gm) : 0.f) + (Ms > -CUDART_INF_F ? Ss * expf(Ms - gm) : 0.f);
        lse = gm + logf(sum);
    }
    const int chosen = S.besti[0];
    const bool at_limit = (n + 1 >= cfg.sample_len || nt + 1 > cfg.n_ctx);
    float* f1 = full_b != nullptr ? full_b + (rows_only ? 0 : (int64_t)n * V) : nullptr;
    float* f2 = (last_full_b != nullptr && at_limit && !rows_only) ? last_full_b : nullptr;
    if (f1 != nullptr || f2 != nullptr) {
        for (int v = threadIdx.x; v < V; v += T) {
            const bool ok = !__ldg(suppress + v) && !(first && __ldg(blank + v)) && range_ok(v) && !(only_ts && v < tsb);
            const float lp = ok ? x[v] - lse : -CUDART_INF_F;
            if (f1) f1[v] = lp;
            if (f2) f2[v] = lp;
        }
    }
    if (threadIdx.x == 0 && !rows_only) {
        logprobs_b[n] = S.best[0] - lse;
        if (chosen == eot) {
            *done_b = 1;
        } else {
            tk[nt] = chosen;
            *n_tokens_b = nt + 1;
            if (at_limit) *done_b = 2;                       // decoding limit reached
        }
    }
}

}  // namespace wts
