// Model-forward operators other than the GEMM: format conversion, LayerNorm, row softmax, log-mel
// pre/post kernels, window gather, token embedding, ragged decoder attention (with the alignment
// heads' pre-softmax rows written straight into the alignment buffer), KV-cache append, and the
// fused logit-filter / log-softmax / greedy-argmax step.  See include/wts.h for the reference
// interfaces each entry replaces.
#include "decode_common.cuh"

namespace wts {

// ------------------------------------------------------------------------------------------ to_sb16
__global__ void to_sb16_kernel(const float* __restrict__ x, int64_t n, __nv_bfloat16* __restrict__ hi,
                               __nv_bfloat16* __restrict__ lo)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        __nv_bfloat16 h, l;
        split_bf16(x[i], h, l);
        hi[i] = h;
        lo[i] = l;
    }
}

// ---------------------------------------------------------------------------------------- layernorm
// one CTA (128 threads) per row; float32 statistics (mean, biased variance), eps = 1e-5.  The row is read once
// into registers (D <= 2048), two block reductions, one write: a single memory round trip per LayerNorm.
constexpr int LN_THREADS = 128, LN_MAXV = 16;
__global__ void __launch_bounds__(LN_THREADS)
layernorm_kernel(const float* x, int64_t ldx, const float* gamma,
                 const float* beta, int M, int D, __nv_bfloat16* o, int64_t ldo,
                 int64_t o_plane, float* of, int64_t ldf)
{
    pdl_launch();
    pdl_wait();
    __shared__ float red[32];
    const int row = blockIdx.x;
    const float* xr = x + (int64_t)row * ldx;
    float v[LN_MAXV];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < LN_MAXV; ++k) {
        const int c = threadIdx.x + LN_THREADS * k;
        v[k] = c < D ? xr[c] : 0.f;
        s += v[k];
    }
    const float mean = block_reduce_sum(s, red) / (float)D;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < LN_MAXV; ++k) {
        const int c = threadIdx.x + LN_THREADS * k;
        const float d = c < D ? v[k] - mean : 0.f;
        q += d * d;
    }
    const float rstd = 1.0f / sqrtf(block_reduce_sum(q, red) / (float)D + 1e-5f);
#pragma unroll
    for (int k = 0; k < LN_MAXV; ++k) {
        const int c = threadIdx.x + LN_THREADS * k;
        if (c < D) {
            const float y = (v[k] - mean) * rstd * gamma[c] + beta[c];
            if (o) {
                __nv_bfloat16 h, l;
                split_bf16(y, h, l);
                o[(int64_t)row * ldo + c] = h;
                o[(int64_t)row * ldo + c + o_plane] = l;
            }
            if (of) of[(int64_t)row * ldf + c] = y;
        }
    }
}

// ------------------------------------------------------------------------------------- softmax rows
// one warp per row, n <= 2048; scores float32 -> probabilities SB16
__global__ void __launch_bounds__(128)
softmax_rows_kernel(const float* __restrict__ s, int64_t lds, int64_t rows, int n,
                    __nv_bfloat16* __restrict__ o, int64_t ldo, int64_t o_plane)
{
    const int64_t row = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float* sr = s + row * lds;
    float v[64];
    float mx = -CUDART_INF_F;
#pragma unroll
    for (int k = 0; k < 64; ++k) {
        const int c = lane + 32 * k;
        v[k] = c < n ? sr[c] : -CUDART_INF_F;
        mx = fmaxf(mx, v[k]);
    }
    mx = warp_max(mx);
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < 64; ++k) {
        v[k] = expf(v[k] - mx);
        sum += v[k];
    }
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
#pragma unroll
    for (int k = 0; k < 64; ++k) {
        const int c = lane + 32 * k;
        if (c < n) {
            __nv_bfloat16 h, l;
            split_bf16(v[k] * inv, h, l);
            o[row * ldo + c] = h;
            o[row * ldo + c + o_plane] = l;
        }
    }
}

// ------------------------------------------------------------------------------------------ log-mel
// frames: Hann(400, periodic) * reflect-padded audio, hop 160; float32 out [n_frames, 400]
__global__ void frames_kernel(const float* __restrict__ audio, int64_t n_samples, int64_t n_total,
                              int64_t n_frames, float* __restrict__ out)
{
    const int64_t t = blockIdx.x;
    if (t >= n_frames) return;
    for (int n = threadIdx.x; n < 400; n += blockDim.x) {
        int64_t i = t * 160 - 200 + n;
        if (i < 0) i = -i;
        if (i >= n_total) i = 2 * (n_total - 1) - i;
        const float x = (i >= 0 && i < n_samples) ? audio[i] : 0.f;
        const float w = 0.5f - 0.5f * cospif((float)n / 200.0f);
        out[t * 400 + n] = x * w;
    }
}

// power: y [n_frames, 2*208] (re | im) -> p [n_frames, 208]
__global__ void power_kernel(const float* __restrict__ y, int64_t ldy, int64_t n_frames, float* __restrict__ p,
                             int64_t ldp)
{
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_frames * 208) return;
    const int64_t t = i / 208;
    const int k = (int)(i - t * 208);
    const float re = y[t * ldy + k], im = y[t * ldy + 208 + k];
    p[t * ldp + k] = re * re + im * im;
}

__device__ __forceinline__ float mel_log10(float m) { return log10f(fmaxf(m, 1e-10f)); }

__global__ void logmel_max_kernel(const float* __restrict__ m, int64_t n, float* __restrict__ out)
{
    __shared__ float red[32];
    float mx = -CUDART_INF_F;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        mx = fmaxf(mx, mel_log10(m[i]));
    mx = block_reduce_max(mx, red);
    if (threadIdx.x == 0) {
        // float max via int ordering (values may be negative): atomicMax on the monotone key
        int key = __float_as_int(mx);
        key = key >= 0 ? key : key ^ 0x7fffffff;
        atomicMax(reinterpret_cast<int*>(out), key);
    }
}

__global__ void logmel_finish_kernel(const float* __restrict__ m, int64_t n, const float* __restrict__ mxkey,
                                     float* __restrict__ out)
{
    int key = *reinterpret_cast<const int*>(mxkey);
    key = key >= 0 ? key : key ^ 0x7fffffff;
    const float gmax = __int_as_float(key);
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float x = mel_log10(m[i]);
        x = fmaxf(x, gmax - 8.0f);
        out[i] = (x + 4.0f) / 4.0f;
    }
}

// window gather: conv1 input [B, 3002, n_mels] SB16, rows 0 and 3001 zero, frames >= size zero
__global__ void window_gather_kernel(const int64_t* __restrict__ mel_ptr, int n_mels,
                                     const int32_t* __restrict__ seek, const int32_t* __restrict__ size, int B,
                                     __nv_bfloat16* __restrict__ out, int64_t o_plane)
{
    const int b = blockIdx.y;
    const float* mel = reinterpret_cast<const float*>(mel_ptr[b]);
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t per = (int64_t)3002 * n_mels;
    if (i >= per) return;
    const int r = (int)(i / n_mels), c = (int)(i - (int64_t)r * n_mels);
    float v = 0.f;
    const int t = r - 1;
    if (t >= 0 && t < size[b]) v = mel[((int64_t)seek[b] + t) * n_mels + c];
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    out[b * per + i] = h;
    out[b * per + i + o_plane] = l;
}

// ------------------------------------------------------------------------------------------- embed
__global__ void embed_kernel(const int32_t* tokens, const int32_t* positions,
                             const float* emb, const float* pos, int rows, int D,
                             float* out)
{
    pdl_launch();
    pdl_wait();
    const int r = blockIdx.x;
    if (r >= rows) return;
    const float* e = emb + (int64_t)tokens[r] * D;
    const float* p = pos + (int64_t)positions[r] * D;
    for (int c = threadIdx.x; c < D; c += blockDim.x) out[(int64_t)r * D + c] = e[c] + p[c];
}

__global__ void gather_rows_kernel(const float* __restrict__ x, int64_t ldx, const int32_t* __restrict__ idx,
                                   int rows, int D, float* __restrict__ out)
{
    const int r = blockIdx.x;
    if (r >= rows) return;
    const float* s = x + (int64_t)idx[r] * ldx;
    for (int c = threadIdx.x; c < D; c += blockDim.x) out[(int64_t)r * D + c] = s[c];
}

// ----------------------------------------------------------------------------- decoder attention
// One CTA (128 threads) per (query row, head); head_dim 64.  Scores, softmax and weighted sum in fp32.
constexpr int DA_THREADS = 128;
__global__ void __launch_bounds__(DA_THREADS)
decoder_attention_kernel(const int kind, const float* q, int64_t ldq, const float* kc,
                         const float* vc, int64_t seq_stride, int ctx,
                         const int32_t* row_seq, const int32_t* row_pos, int H,
                         __nv_bfloat16* o, int64_t ldo, int64_t o_plane, float* qk_out,
                         const int32_t* head_slot, int n_slots, int qk_rows,
                         const int32_t* qk_row, const int32_t* row_active)
{
    pdl_launch();
    pdl_wait();
    extern __shared__ float sm[];
    float* sc = sm;                 // [ctx] scores
    float* qs = sm + ctx;           // [64]
    float* red = qs + 64;           // [32]
    float* part = red + 32;         // [2][64]
    const int r = blockIdx.x, h = blockIdx.y;
    if (row_active != nullptr && !row_active[r]) return;
    const int seq = row_seq[r];
    const int nk = kind == 1 ? ctx : row_pos[r] + 1;
    const float* K = kc + (int64_t)seq * seq_stride + (int64_t)h * ctx * 64;
    const float* V = vc + (int64_t)seq * seq_stride + (int64_t)h * ctx * 64;
    if (kind == 2) {
        // decode step (one row per sequence): q points at packed [q | k | v] rows; this CTA appends its head's K/V
        // of the new position to the cache itself (saves the separate kv_append launch).  The barrier below makes
        // the two 64-float rows visible to the whole CTA before the score loop reads position row_pos[r].
        const float* src = q + (int64_t)r * ldq + h * 64;
        const int64_t at = (int64_t)(nk - 1) * 64 + (threadIdx.x & 63);
        if (threadIdx.x < 64) const_cast<float*>(K)[at] = src[(int64_t)H * 64 + threadIdx.x];
        else                  const_cast<float*>(V)[at] = src[(int64_t)2 * H * 64 + (threadIdx.x & 63)];
    }
    if (threadIdx.x < 64) qs[threadIdx.x] = q[(int64_t)r * ldq + h * 64 + threadIdx.x];
    __syncthreads();
    float mx = -CUDART_INF_F;
    for (int j = threadIdx.x; j < nk; j += DA_THREADS) {
        const float4* kr = reinterpret_cast<const float4*>(K + (int64_t)j * 64);
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < 16; ++c) {
            const float4 kv = kr[c];
            acc += qs[4 * c] * kv.x + qs[4 * c + 1] * kv.y + qs[4 * c + 2] * kv.z + qs[4 * c + 3] * kv.w;
        }
        sc[j] = acc;
        mx = fmaxf(mx, acc);
    }
    __syncthreads();
    if (kind == 1 && qk_out != nullptr) {
        const int slot = head_slot[h];
        const int qr = qk_row[r];
        if (slot >= 0 && qr >= 0) {
            float* dst = qk_out + (((int64_t)seq * n_slots + slot) * qk_rows + qr) * (int64_t)ctx;
            for (int j = threadIdx.x; j < nk; j += DA_THREADS) dst[j] = sc[j];
        }
    }
    mx = block_reduce_max(mx, red);
    float sum = 0.f;
    for (int j = threadIdx.x; j < nk; j += DA_THREADS) {
        const float e = expf(sc[j] - mx);
        sc[j] = e;
        sum += e;
    }
    sum = block_reduce_sum(sum, red);
    const float inv = 1.0f / sum;
    const int c = threadIdx.x & 63, g = threadIdx.x >> 6;
    float acc = 0.f;
    for (int j = g; j < nk; j += 2) acc += sc[j] * V[(int64_t)j * 64 + c];
    part[g * 64 + c] = acc;
    __syncthreads();
    if (threadIdx.x < 64) {
        const float y = (part[threadIdx.x] + part[64 + threadIdx.x]) * inv;
        __nv_bfloat16 hi, lo;
        split_bf16(y, hi, lo);
        o[(int64_t)r * ldo + h * 64 + threadIdx.x] = hi;
        o[(int64_t)r * ldo + h * 64 + threadIdx.x + o_plane] = lo;
    }
}


// -------------------------------------------------------------- cross attention, fp16 K/V caches
// Decode-time cross-attention is a pure HBM stream of the window's K/V (1500 x 64 per head); storing
// them in fp16 halves that stream.  Measured on the CPU oracle: fp16 K+V shift the logits by < 3e-4 but
// the exported scores by 2.6e-3, so the ALIGNMENT heads keep a float32 copy of K (their pre-softmax
// rows are the DTW input and must stay within 1e-3 of the reference); all other heads use fp16 K.
__global__ void cross_kv_pack_kernel(const float* __restrict__ src, __half* __restrict__ dst16,
                                     float* __restrict__ dst_align, const int32_t* __restrict__ head_slot,
                                     int s0, int n_l, int H, int ctx)
{
    const int bh = blockIdx.x;                      // b * H + h
    const int b = bh / H, h = bh - b * H;
    const float* s = src + (int64_t)bh * ctx * 64;
    __half* d = dst16 + (int64_t)bh * ctx * 64;
    const int slot = dst_align ? head_slot[h] : -1;
    float* da = slot >= 0 ? dst_align + ((int64_t)b * n_l + slot - s0) * ctx * 64 : nullptr;
    for (int i = threadIdx.x; i < ctx * 64; i += blockDim.x) {
        const float v = s[i];
        d[i] = __float2half_rn(v);
        if (da) da[i] = v;
    }
}

// (The decode-step kernels take plain, not __restrict__, pointers: under programmatic dependent launch a consumer is
// resident before its producer has finished, so producer-written buffers must not be read through the non-coherent
// ld.global.nc path the compiler picks for const __restrict__ data.)
// One CTA per (query row, head): decode_common.cuh ca_row_head (one pass, online softmax, K/V streamed once).
__global__ void __launch_bounds__(CA_THREADS)
cross_attention_f16_kernel(const float* q, int64_t ldq, const __half* k16,
                           const __half* v16, const float* k_align,
                           const int32_t* head_slot, int n_slots, int s0, int n_l, int ctx,
                           const int32_t* row_seq, int H, __nv_bfloat16* o, int64_t ldo,
                           int64_t o_plane, float* qk_out, int qk_rows, const int32_t* qk_row,
                           const int32_t* row_active)
{
    pdl_launch();
    pdl_wait();
    __shared__ CaScratch sc;
    const int r = blockIdx.x, h = blockIdx.y;
    if (row_active != nullptr && !row_active[r]) return;   // finished sequence: skip its K/V stream
    const int seq = row_seq[r];
    const int slot = head_slot[h];
    const int c8 = threadIdx.x & 7;
    float qf[8];
    {
        const float4* qp = reinterpret_cast<const float4*>(q + (int64_t)r * ldq + h * 64 + c8 * 8);
        const float4 a = qp[0], b = qp[1];
        qf[0] = a.x; qf[1] = a.y; qf[2] = a.z; qf[3] = a.w; qf[4] = b.x; qf[5] = b.y; qf[6] = b.z; qf[7] = b.w;
    }
    const __half* V = v16 + ((int64_t)seq * H + h) * ctx * 64;
    float* qk_dst = nullptr;
    const float* kal = nullptr;
    if (slot >= 0) {
        kal = k_align + ((int64_t)seq * n_l + slot - s0) * ctx * 64;
        if (qk_out != nullptr) {
            const int qr = qk_row[r];
            if (qr >= 0) qk_dst = qk_out + (((int64_t)seq * n_slots + slot) * qk_rows + qr) * (int64_t)ctx;
        }
    }
    const float y = ca_row_head<4>(qf, k16 + ((int64_t)seq * H + h) * ctx * 64, V, kal, qk_dst, ctx, sc);
    if (threadIdx.x < 64) {
        __nv_bfloat16 hi, lo;
        split_bf16(y, hi, lo);
        o[(int64_t)r * ldo + h * 64 + threadIdx.x] = hi;
        o[(int64_t)r * ldo + h * 64 + threadIdx.x + o_plane] = lo;
    }
}

__global__ void kv_append_kernel(const float* k, const float* v, int64_t ld,
                                 const int32_t* row_seq, const int32_t* row_pos, int H,
                                 int ctx, float* kc, float* vc, int64_t seq_stride)
{
    pdl_launch();
    pdl_wait();
    const int r = blockIdx.x;
    const int seq = row_seq[r], pos = row_pos[r];
    for (int c = threadIdx.x; c < H * 64; c += blockDim.x) {
        const int h = c >> 6, d = c & 63;
        const int64_t dst = (int64_t)seq * seq_stride + ((int64_t)h * ctx + pos) * 64 + d;
        kc[dst] = k[(int64_t)r * ld + c];
        vc[dst] = v[(int64_t)r * ld + c];
    }
}

// ------------------------------------------------------------------------------------ decode select
// one CTA per sequence: decode_common.cuh select_row
constexpr int DS_THREADS = 1024;
__global__ void __launch_bounds__(DS_THREADS)
decode_select_kernel(float* logits, int64_t ldl, const WtsDecodeCfg cfg,
                     const uint8_t* suppress, const uint8_t* blank,
                     int32_t* tokens, int32_t* n_tokens,
                     const int32_t* n_prompt, int32_t* done,
                     float* logprobs, int lp_ld, float* full, float* last_full)
{
    pdl_launch();
    pdl_wait();
    __shared__ SelectScratch S;
    const int b = blockIdx.x;
    if (done[b]) return;
    select_row(logits + (int64_t)b * ldl, cfg, suppress, blank, tokens + (int64_t)b * cfg.tokens_ld, n_tokens + b,
               n_prompt[b], done + b, logprobs + (int64_t)b * lp_ld,
               full != nullptr ? full + (int64_t)b * lp_ld * cfg.n_vocab : nullptr,
               last_full != nullptr ? last_full + (int64_t)b * cfg.n_vocab : nullptr, S);
}

// filtered log-softmax rows only (beam search / sampling): one CTA per sequence, no state update
__global__ void __launch_bounds__(DS_THREADS)
filtered_logprobs_kernel(const float* logits, int64_t ldl, const WtsDecodeCfg cfg, const uint8_t* suppress, const uint8_t* blank,
                         int32_t* tokens, int32_t* n_tokens, const int32_t* n_prompt, float* out)
{
    __shared__ SelectScratch S;
    const int b = blockIdx.x;
    select_row(logits + (int64_t)b * ldl, cfg, suppress, blank, tokens + (int64_t)b * cfg.tokens_ld, n_tokens + b,
               n_prompt[b], nullptr, nullptr, out + (int64_t)b * cfg.n_vocab, nullptr, S, true);
}

__global__ void step_inputs_kernel(const int32_t* tokens, int ld, const int32_t* n_tokens,
                                   const int32_t* n_prompt, const int32_t* done, int B,
                                   int32_t* tok, int32_t* pos, int32_t* qk_row,
                                   int32_t* active)
{
    pdl_launch();
    pdl_wait();
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int nt = n_tokens[b];
    tok[b] = tokens[(int64_t)b * ld + nt - 1];
    pos[b] = nt - 1;
    qk_row[b] = done[b] ? -1 : nt - n_prompt[b];
    if (active) active[b] = done[b] ? 0 : 1;
}

__global__ void softmax_pick_kernel(const float* __restrict__ logits, int64_t ldl, int n, int index,
                                    float* __restrict__ out)
{
    __shared__ float red[32];
    const float* x = logits + (int64_t)blockIdx.x * ldl;
    float mx = -CUDART_INF_F;
    for (int v = threadIdx.x; v < n; v += blockDim.x) mx = fmaxf(mx, x[v]);
    mx = block_reduce_max(mx, red);
    float s = 0.f;
    for (int v = threadIdx.x; v < n; v += blockDim.x) s += expf(x[v] - mx);
    s = block_reduce_sum(s, red);
    if (threadIdx.x == 0) out[blockIdx.x] = expf(x[index] - mx) / s;
}

// log_softmax(logits[row[i]])[token[i]] for a list of (row, token) pairs: the teacher-forced log-probabilities the
// two-pass ("naive") strategy turns into word confidences (T.py:1245-1246, 1285-1300).  One CTA per pair.
__global__ void logprob_gather_kernel(const float* logits, int64_t ldl, int n, const int32_t* rows, const int32_t* tokens,
                                      float* out)
{
    __shared__ float red[32];
    const float* x = logits + (int64_t)rows[blockIdx.x] * ldl;
    float mx = -CUDART_INF_F;
    for (int v = threadIdx.x; v < n; v += blockDim.x) mx = fmaxf(mx, x[v]);
    mx = block_reduce_max(mx, red);
    float s = 0.f;
    for (int v = threadIdx.x; v < n; v += blockDim.x) s += expf(x[v] - mx);
    s = block_reduce_sum(s, red);
    if (threadIdx.x == 0) out[blockIdx.x] = (x[tokens[blockIdx.x]] - mx) - logf(s);
}

}  // namespace wts

using namespace wts;

static inline int grid_for(int64_t n, int block, int cap = 132 * 16)
{
    int64_t g = (n + block - 1) / block;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

extern "C" int wts_to_sb16(const float* d_x, int64_t n, void* d_hi, void* d_lo, void* stream)
{
    if (n <= 0) return 0;
    to_sb16_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(d_x, n, (__nv_bfloat16*)d_hi, (__nv_bfloat16*)d_lo);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_layernorm(const float* d_x, int64_t ldx, const float* d_gamma, const float* d_beta, int32_t M,
                             int32_t D, void* d_out_sb16, int64_t ldo, int64_t o_plane, float* d_out_f32,
                             int64_t ldf, void* stream)
{
    if (M <= 0) return 0;
    if (D > LN_THREADS * LN_MAXV) { set_error("wts_layernorm: D=%d > %d", D, LN_THREADS * LN_MAXV); return -2; }
    WTS_CUDA_CHECK(launch_pdl(layernorm_kernel, dim3(M), dim3(LN_THREADS), 0, (cudaStream_t)stream, d_x, ldx, d_gamma, d_beta, M, D,
                                                                   (__nv_bfloat16*)d_out_sb16, ldo, o_plane, d_out_f32, ldf));
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_softmax_rows(const float* d_s, int64_t lds, int64_t rows, int32_t n, void* d_out_sb16,
                                int64_t ldo, int64_t o_plane, void* stream)
{
    if (rows <= 0) return 0;
    if (n > 2048) { set_error("wts_softmax_rows: n=%d > 2048", n); return -2; }
    softmax_rows_kernel<<<(unsigned)((rows + 3) / 4), 128, 0, (cudaStream_t)stream>>>(d_s, lds, rows, n,
                                                                                     (__nv_bfloat16*)d_out_sb16, ldo, o_plane);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_frames(const float* d_audio, int64_t n_samples, int64_t n_total, int64_t n_frames, void* d_out,
                          int64_t o_plane, void* stream)
{
    (void)o_plane;
    if (n_frames <= 0) return 0;
    frames_kernel<<<(unsigned)n_frames, 128, 0, (cudaStream_t)stream>>>(d_audio, n_samples, n_total, n_frames, (float*)d_out);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_power(const float* d_y, int64_t ldy, int64_t n_frames, void* d_out, int64_t ldo, int64_t o_plane,
                         void* stream)
{
    (void)o_plane;
    if (n_frames <= 0) return 0;
    power_kernel<<<(unsigned)((n_frames * 208 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_y, ldy, n_frames, (float*)d_out, ldo);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_logmel_max(const float* d_m, int64_t n, float* d_max, void* stream)
{
    // d_max must be pre-set by the caller to the key of -inf (0x807fffff ^ 0x7fffffff = int min side): use -FLT_MAX key
    logmel_max_kernel<<<grid_for(n, 256, 1024), 256, 0, (cudaStream_t)stream>>>(d_m, n, d_max);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_logmel_finish(const float* d_m, int64_t n_frames, int32_t n_mels, const float* d_max,
                                 float* d_out_f32, void* stream)
{
    const int64_t n = n_frames * n_mels;
    logmel_finish_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(d_m, n, d_max, d_out_f32);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_window_gather(const int64_t* d_mel_ptr, int32_t n_mels, const int32_t* d_seek,
                                 const int32_t* d_size, int32_t B, void* d_out, int64_t o_plane, void* stream)
{
    if (B <= 0) return 0;
    dim3 grid((unsigned)(((int64_t)3002 * n_mels + 255) / 256), B);
    window_gather_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(d_mel_ptr, n_mels, d_seek, d_size, B,
                                                                 (__nv_bfloat16*)d_out, o_plane);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_embed(const int32_t* d_tokens, const int32_t* d_positions, const float* d_emb, const float* d_pos,
                         int32_t rows, int32_t D, float* d_out, void* stream)
{
    if (rows <= 0) return 0;
    WTS_CUDA_CHECK(launch_pdl(embed_kernel, dim3(rows), dim3(256), 0, (cudaStream_t)stream, d_tokens, d_positions, d_emb, d_pos, rows, D, d_out));
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_gather_rows(const float* d_x, int64_t ldx, const int32_t* d_idx, int32_t rows, int32_t D,
                               float* d_out, void* stream)
{
    if (rows <= 0) return 0;
    gather_rows_kernel<<<rows, 256, 0, (cudaStream_t)stream>>>(d_x, ldx, d_idx, rows, D, d_out);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_decoder_attention(int32_t kind, const float* d_q, int64_t ldq, const float* d_k, const float* d_v,
                                     int64_t seq_stride, int32_t ctx, const int32_t* d_row_seq,
                                     const int32_t* d_row_pos, int32_t rows, int32_t H, void* d_out_sb16, int64_t ldo,
                                     int64_t o_plane, float* d_qk_out, const int32_t* d_head_slot, int32_t n_slots,
                                     int32_t qk_rows, const int32_t* d_qk_row, const int32_t* d_row_active, void* stream)
{
    if (rows <= 0) return 0;
    const size_t smem = ((size_t)ctx + 64 + 32 + 128) * sizeof(float);
    dim3 grid(rows, H);
    WTS_CUDA_CHECK(launch_pdl(decoder_attention_kernel, grid, dim3(DA_THREADS), smem, (cudaStream_t)stream, 
        kind, d_q, ldq, d_k, d_v, seq_stride, ctx, d_row_seq, d_row_pos, H, (__nv_bfloat16*)d_out_sb16, ldo, o_plane,
        d_qk_out, d_head_slot, n_slots, qk_rows, d_qk_row, d_row_active));
    WTS_LAUNCH_CHECK();
    return 0;
}


extern "C" int wts_cross_kv_pack_layer(const float* d_src, void* d_dst16, float* d_dst_align,
                                       const int32_t* d_head_slot, int32_t align_s0, int32_t align_n, int32_t B,
                                       int32_t H, int32_t ctx, void* stream)
{
    if (B <= 0) return 0;
    cross_kv_pack_kernel<<<B * H, 256, 0, (cudaStream_t)stream>>>(d_src, (__half*)d_dst16, d_dst_align, d_head_slot,
                                                                 align_s0, align_n, H, ctx);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_cross_kv_pack(const float* d_src, void* d_dst16, float* d_dst_align, const int32_t* d_head_slot,
                                 int32_t n_slots, int32_t B, int32_t H, int32_t ctx, void* stream)
{
    return wts_cross_kv_pack_layer(d_src, d_dst16, d_dst_align, d_head_slot, 0, n_slots, B, H, ctx, stream);
}

extern "C" int wts_cross_attention_f16_layer(const float* d_q, int64_t ldq, const void* d_k16, const void* d_v16,
                                             const float* d_k_align, const int32_t* d_head_slot, int32_t n_slots,
                                             int32_t align_s0, int32_t align_n, int32_t ctx, const int32_t* d_row_seq,
                                             int32_t rows, int32_t H, void* d_out_sb16, int64_t ldo, int64_t o_plane,
                                             float* d_qk_out, int32_t qk_rows, const int32_t* d_qk_row,
                                             const int32_t* d_row_active, void* stream)
{
    if (rows <= 0) return 0;
    if ((ldq & 3) || (reinterpret_cast<uintptr_t>(d_q) & 15)) { set_error("wts_cross_attention_f16: q must be 16-byte aligned"); return -2; }
    dim3 grid(rows, H);
    WTS_CUDA_CHECK(launch_pdl(cross_attention_f16_kernel, grid, dim3(CA_THREADS), 0, (cudaStream_t)stream, 
        d_q, ldq, (const __half*)d_k16, (const __half*)d_v16, d_k_align, d_head_slot, n_slots, align_s0, align_n, ctx,
        d_row_seq, H, (__nv_bfloat16*)d_out_sb16, ldo, o_plane, d_qk_out, qk_rows, d_qk_row, d_row_active));
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_cross_attention_f16(const float* d_q, int64_t ldq, const void* d_k16, const void* d_v16,
                                       const float* d_k_align, const int32_t* d_head_slot, int32_t n_slots,
                                       int32_t ctx, const int32_t* d_row_seq, int32_t rows, int32_t H,
                                       void* d_out_sb16, int64_t ldo, int64_t o_plane, float* d_qk_out,
                                       int32_t qk_rows, const int32_t* d_qk_row, const int32_t* d_row_active,
                                       void* stream)
{
    return wts_cross_attention_f16_layer(d_q, ldq, d_k16, d_v16, d_k_align, d_head_slot, n_slots, 0, n_slots, ctx,
                                         d_row_seq, rows, H, d_out_sb16, ldo, o_plane, d_qk_out, qk_rows, d_qk_row,
                                         d_row_active, stream);
}

extern "C" int wts_kv_append(const float* d_k, const float* d_v, int64_t ld, const int32_t* d_row_seq,
                             const int32_t* d_row_pos, int32_t rows, int32_t H, int32_t ctx, float* d_kc, float* d_vc,
                             int64_t seq_stride, void* stream)
{
    if (rows <= 0) return 0;
    WTS_CUDA_CHECK(launch_pdl(kv_append_kernel, dim3(rows), dim3(256), 0, (cudaStream_t)stream, d_k, d_v, ld, d_row_seq, d_row_pos, H, ctx, d_kc, d_vc, seq_stride));
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_decode_select(float* d_logits, int64_t ldl, const WtsDecodeCfg* cfg, const uint8_t* d_suppress,
                                 const uint8_t* d_blank, int32_t* d_tokens, int32_t* d_n_tokens,
                                 const int32_t* d_n_prompt, int32_t* d_done, float* d_logprobs, int32_t lp_ld,
                                 float* d_full_logprobs, float* d_last_full, int32_t B, void* stream)
{
    if (B <= 0) return 0;
    WTS_CUDA_CHECK(launch_pdl(decode_select_kernel, dim3(B), dim3(DS_THREADS), 0, (cudaStream_t)stream, d_logits, ldl, *cfg, d_suppress, d_blank, d_tokens,
                                                                    d_n_tokens, d_n_prompt, d_done, d_logprobs, lp_ld,
                                                                    d_full_logprobs, d_last_full));
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_filtered_logprobs(const float* d_logits, int64_t ldl, const WtsDecodeCfg* cfg, const uint8_t* d_suppress,
                                     const uint8_t* d_blank, int32_t* d_tokens, int32_t* d_n_tokens, const int32_t* d_n_prompt,
                                     float* d_out, int32_t B, void* stream)
{
    if (B <= 0) return 0;
    if (!d_logits || !cfg || !d_suppress || !d_blank || !d_tokens || !d_n_tokens || !d_n_prompt || !d_out) {
        set_error("wts_filtered_logprobs: null pointer");
        return -2;
    }
    filtered_logprobs_kernel<<<B, DS_THREADS, 0, (cudaStream_t)stream>>>(d_logits, ldl, *cfg, d_suppress, d_blank, d_tokens,
                                                                         d_n_tokens, d_n_prompt, d_out);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_step_inputs(const int32_t* d_tokens, int32_t tokens_ld, const int32_t* d_n_tokens,
                               const int32_t* d_n_prompt, const int32_t* d_done, int32_t B, int32_t* d_tok,
                               int32_t* d_pos, int32_t* d_qk_row, int32_t* d_active, void* stream)
{
    if (B <= 0) return 0;
    WTS_CUDA_CHECK(launch_pdl(step_inputs_kernel, dim3((B + 127) / 128), dim3(128), 0, (cudaStream_t)stream, d_tokens, tokens_ld, d_n_tokens, d_n_prompt,
                                                                         d_done, B, d_tok, d_pos, d_qk_row, d_active));
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_softmax_pick(const float* d_logits, int64_t ldl, int32_t n, int32_t index, float* d_out,
                                int32_t rows, void* stream)
{
    if (rows <= 0) return 0;
    softmax_pick_kernel<<<rows, 512, 0, (cudaStream_t)stream>>>(d_logits, ldl, n, index, d_out);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_logprob_gather(const float* d_logits, int64_t ldl, int32_t n, const int32_t* d_rows,
                                  const int32_t* d_tokens, float* d_out, int32_t count, void* stream)
{
    if (count <= 0) return 0;
    if (!d_logits || !d_rows || !d_tokens || !d_out) { set_error("wts_logprob_gather: null pointer"); return -2; }
    logprob_gather_kernel<<<count, 512, 0, (cudaStream_t)stream>>>(d_logits, ldl, n, d_rows, d_tokens, d_out);
    WTS_LAUNCH_CHECK();
    return 0;
}
