/*
 * libwts — C-ABI of the H100-native word-alignment hot path of whisper-timestamped.
 *
 * Conventions (all entry points):
 *   - every pointer named d_* is a DEVICE pointer owned by the caller (PyTorch allocations are
 *     only the memory carrier); the library never frees or retains it past the call, except
 *     the persistent objects created by *_create and freed by *_destroy;
 *   - `stream` is a cudaStream_t passed as void*; work is enqueued asynchronously on it;
 *   - return value: 0 = OK, <0 = error (message via wts_last_error(), thread-local);
 *   - no C++ exception crosses the ABI; there is no CPU fallback: if no sm_90a device code can
 *     run, the call fails with an error.
 *
 * Each entry cites the reference interface it replaces
 * (T.py = /root/reference/whisper_timestamped/transcribe.py).
 */
#ifndef WTS_H
#define WTS_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WTS_VERSION 103
#define WTS_SEG_NONPOSITIVE 1
#define WTS_SEG_PITCH16 2

/* One alignment problem (= one speech segment handed to perform_word_alignment, T.py:1428).
 * Built on the host, copied to the device by the caller, consumed by the kernels. */
typedef struct WtsSegDesc {
    int32_t window;    /* which decoded 30-s window of the qk buffer the rows live in            */
    int32_t row0;      /* first token row inside that window's qk rows                          */
    int32_t last_row;  /* row used for the LAST token (normally row0+T-1; differs when the text
                          is truncated because T > F, T.py:1516-1535)                           */
    int32_t T;         /* number of tokens (rows of the cost matrix)                            */
    int32_t f0;        /* start_token: first encoder frame of the slice (T.py:1540)             */
    int32_t F;         /* number of frames in the slice (= end_token - start_token)             */
    int32_t max_dur;   /* padding limit in frames (find_start_padding(mfcc)//2, T.py:1556-1558),
                          <=0 when there is no padding                                          */
    int32_t flags;     /* bit 0 (WTS_SEG_NONPOSITIVE): the float32 cost matrix is <= 0 everywhere with
                          cost[0,0] < 0 (true for the output of wts_attn_prep_batch): enables the
                          integer-compare DTW fast path.
                          bit 1 (WTS_SEG_PITCH16): rows of the cost matrix are padded to 16 bytes, i.e. the
                          row pitch is (F + 3) & ~3 elements instead of F (padding columns hold zeros): lets
                          the DTW kernel stage rows with 16-byte bulk copies                      */
    int64_t cost_off;  /* element offset of this segment's [T,F] matrix in the cost buffer      */
    int64_t jumps_off; /* element offset of this segment's T+1 jumps in the jumps buffer        */
    int64_t dir_off;   /* uint32 offset of this segment's direction words in the DTW workspace  */
    int64_t bnd_off;   /* float64 offset of the strip-boundary row in the DTW workspace
                          (only read when T > 32)                                               */
} WtsSegDesc;

int         wts_version(void);
const char* wts_last_error(void);

/* Workspace sizing helpers for wts_dtw_batch (pure host arithmetic).
 * dir words (uint32) and boundary doubles one segment of T tokens x F frames needs. */
int64_t wts_dtw_dir_words(int32_t T, int32_t F);
int64_t wts_dtw_bnd_doubles(int32_t T, int32_t F);

/*
 * Fused attention post-processing — replaces T.py:1540-1568
 *   (slice frames, stack alignment heads, scipy.ndimage.median_filter(1,1,9), softmax over
 *    frames, mean over heads, / L2-norm over tokens, negate, padding mask, cost[0,0]=min).
 * d_qk:   float32 [n_windows, N, Tmax, Fmax] pre-softmax cross-attention rows of the N selected
 *         alignment heads (what hook_attention_weights captures at T.py:783-793), row k = the
 *         row computed with input token k.
 * d_cost: float32 output, matrices back to back at segs[i].cost_off (values are exactly the
 *         float32 numbers the reference widens to float64 at T.py:1550).
 * max_T / max_F: maxima of segs[i].T / segs[i].F over the batch (launch geometry only).
 */
int wts_attn_prep_batch(const float* d_qk, int32_t N, int32_t Tmax, int32_t Fmax,
                        const WtsSegDesc* d_segs, int32_t nseg, int32_t max_T, int32_t max_F,
                        float* d_cost, void* stream);

/* The same with the row kernel chosen: kernel 1 = one warp per token row walks the N heads in order; kernel 2 = one
 * CTA per token row, its warps take disjoint head subsets and their sums are added in warp order (deterministic, but
 * a different float32 summation order than kernel 1); kernel 0 = wts_attn_prep_batch's choice: kernel 2 when
 * N >= WTS_PREP_HEADS_MIN_N, else kernel 1. */
#define WTS_PREP_HEADS_MIN_N 32
int wts_attn_prep_batch_kernel(const float* d_qk, int32_t N, int32_t Tmax, int32_t Fmax,
                               const WtsSegDesc* d_segs, int32_t nseg, int32_t max_T, int32_t max_F,
                               float* d_cost, int32_t kernel, void* stream);

/*
 * Batched monotonic DTW — replaces dtw.dtw(weights, step_pattern=symmetric1) at T.py:1572-1581
 * and the jumps extraction at T.py:1648-1652.
 * d_cost:  float32 (cost_is_f64 == 0) or float64 (cost_is_f64 == 1) local-cost matrices.
 * d_dir_ws: uint32 workspace, segment i uses wts_dtw_dir_words(T,F) words at dir_off.
 * d_bnd_ws: float64 workspace, segment i uses wts_dtw_bnd_doubles(T,F) doubles at bnd_off.
 * d_jumps: int32 output, T+1 entries per segment at jumps_off (first frame of every token row on
 *          the optimal path, then the last frame index).
 * d_path:  optional (may be NULL) int32 output of the full warping path (alignment.index1s /
 *          .index2s): segment i writes index1s at d_path[path_off[i] .. +len) and index2s at
 *          d_path[path_off[i] + T + F .. +len), ascending; len goes to d_path_len[i].
 * d_status: optional int32 per segment, 0 = ok, 1 = non-finite accumulated cost (the reference
 *          raises "No warping path found" in that case).
 */
int wts_dtw_batch(const void* d_cost, int32_t cost_is_f64,
                  const WtsSegDesc* d_segs, int32_t nseg,
                  uint32_t* d_dir_ws, double* d_bnd_ws,
                  int32_t* d_jumps, int32_t* d_path, const int64_t* d_path_off,
                  int32_t* d_path_len, int32_t* d_status, void* stream);

/* Same, with hints about the batch: the largest T / F (0 = unknown; they size the fast paths' shared-memory buffers and
 * row unrolling — segments above the hints still run, in the general kernel) and all_flags = the bitwise AND of
 * WtsSegDesc.flags over the batch (0 = unknown; when every segment is known to belong to a fast path the general kernel
 * is not launched).  Batches of WTS_DTW_LANE_MIN (environment, default 8192) matrices or more use the lane-per-matrix
 * kernel (T <= 32, any F), smaller ones the warp-per-matrix wavefront kernels; results are identical. */
int wts_dtw_batch_sized(const void* d_cost, int32_t cost_is_f64,
                  const WtsSegDesc* d_segs, int32_t nseg,
                  uint32_t* d_dir_ws, double* d_bnd_ws,
                  int32_t* d_jumps, int32_t* d_path, const int64_t* d_path_off,
                  int32_t* d_path_len, int32_t* d_status, int32_t max_T, int32_t max_F, int32_t all_flags,
                  void* stream);

/* detect_disfluencies (T.py:1656-1683): for every token t of every segment, d_out[jumps_off + t] = -1, or — when
 * scipy.signal.find_peaks(-cost[t, jumps[t]:jumps[t+1]], width=3, prominence=0.02) finds more than one peak —
 * round(left_ips[-1]), the offset (from jumps[t]) at which the token really starts.  d_cost / d_segs / d_jumps are
 * the buffers of wts_attn_prep_batch / wts_dtw_batch (float32 costs; descriptors in any order). */
int wts_disfluency_starts(const float* d_cost, const WtsSegDesc* d_segs, int32_t nseg, const int32_t* d_jumps,
                          int32_t* d_out, void* stream);


/* ------------------------------------------------------------------------------------------------
 * Model forward operators (replace the openai-whisper modules the reference drives through
 * model.transcribe / model(mfcc, tokens), T.py:904, 1244, and hooks into at T.py:887-900).
 *
 * "split-bf16" (SB16) is the GEMM operand format of this library: a float32 value x is carried as
 * two bfloat16 planes hi = bf16(x), lo = bf16(x - hi) (16 mantissa bits).  Tensor-core GEMMs form
 * hi*hi + lo*hi + hi*lo in float32 (error-compensated, ~1e-5 relative) so that logits and
 * cross-attention scores stay within the 1e-3 bar against the reference's float32 CPU path.
 * ------------------------------------------------------------------------------------------------ */

typedef struct WtsGemm {
    /* C[z][m][n] = act(alpha * sum_k A[z][m][k] * B[z][n][k] + bias) + residual   (z = zo*batch_inner + zi) */
    const void* a;  int64_t lda, a_plane, a_bo, a_bi;   /* SB16 [M,K]: row stride, hi->lo plane stride, batch strides (elements) */
    const void* b;  int64_t ldb, b_plane, b_bo, b_bi;   /* SB16 [N,K] */
    int32_t M, N, K, batch_outer, batch_inner;
    float alpha;
    const float* bias;        /* [N] (bias_on_m == 0) or [M] (bias_on_m == 1), may be NULL */
    int32_t bias_on_m;
    int32_t act;              /* 0 = none, 1 = exact (erf) GELU */
    const float* residual; int64_t ldr, r_bo, r_bi;     /* float32, may be NULL, may alias out_f32 */
    float* out_f32;   int64_t ldc, c_bo, c_bi;          /* float32 output (may be NULL) */
    void*  out_sb16;  int64_t ldo, o_plane, o_bo, o_bi; /* SB16 output (may be NULL) */
    int32_t head_dim; int64_t head_stride;   /* if head_dim > 0 output column n goes to
                                                (n / head_dim) * head_stride + m * ld + (n % head_dim) */
    int32_t backend;          /* 0 = wgmma tensor cores, 1 = SIMT float32 validator */
    int32_t a_is_f32, b_is_f32;   /* SIMT backend only: operand is plain float32 (log-mel DFT / filterbank GEMMs) */
    const int32_t* row_mask;  /* optional [M] (M <= 128, unbatched): rows with mask 0 are skipped, their outputs stay
                                 untouched (finished windows of a decode batch); NULL = every row */
    int32_t b_const;          /* 1: B is a model weight that no kernel still in flight on the stream writes, so a
                                 decode-time GEMM may start loading B before the previous kernel has completed */
} WtsGemm;

/* Error-compensated GEMM.  Replaces every torch Linear / Conv1d / matmul of the encoder and decoder. */
int wts_gemm(const WtsGemm* g, void* stream);

/* float32 -> SB16 planes (used for weights at load time and for mel / embeddings). */
int wts_to_sb16(const float* d_x, int64_t n, void* d_hi, void* d_lo, void* stream);

/* LayerNorm over the last dim (eps 1e-5, float32 statistics): rows [M, D] float32 -> SB16 and/or f32. */
int wts_layernorm(const float* d_x, int64_t ldx, const float* d_gamma, const float* d_beta, int32_t M,
                  int32_t D, void* d_out_sb16, int64_t ldo, int64_t o_plane, float* d_out_f32, int64_t ldf,
                  void* stream);

/* Row softmax over float32 scores [rows, n] (ld) -> SB16 probabilities (encoder self-attention). */
int wts_softmax_rows(const float* d_s, int64_t lds, int64_t rows, int32_t n, void* d_out_sb16, int64_t ldo,
                     int64_t o_plane, void* stream);

/* Fused encoder self-attention (wgmma): out = softmax(q k^T) v per (window, head), head dim 64; the score matrix
 * stays on the SM (registers / shared memory).  d_qk: SB16 [B*n_ctx, 2D] (q | k, scale already folded in);
 * d_vt: SB16 V^T [B*D, ld_vt] (row = channel, column = key); d_out: SB16 [B*n_ctx, D]. */
int wts_enc_attention(const void* d_qk, int64_t ld_qk, int64_t qk_plane, const void* d_vt, int64_t ld_vt,
                      int64_t vt_plane, int32_t B, int32_t H, int32_t D, int32_t n_ctx, void* d_out, int64_t ldo,
                      int64_t o_plane, void* stream);

/* Log-mel front end — replaces whisper.log_mel_spectrogram (T.py:1213; upstream transcribe()).
 * wts_frames:  audio [n] -> Hann-windowed, reflect-padded frames float32 [n_frames, 400] (hop 160).
 * (DFT as a float32 GEMM against the [2*208, 400] cos|-sin basis, wts_gemm with a_is_f32/b_is_f32.)
 * wts_power:   DFT GEMM output [n_frames, 2*208] (re | im) -> power float32 [n_frames, 208].
 * (mel filterbank as a float32 GEMM.)
 * wts_logmel_max / wts_logmel_finish: mel energies [n_frames, n_mels] -> log10(clamp 1e-10), floor at
 *              (global max - 8), (x+4)/4; time-major float32 [n_frames, n_mels].  d_max holds an order-
 *              preserving int key and must be initialised to INT32_MIN by the caller. */
int wts_frames(const float* d_audio, int64_t n_samples, int64_t n_total, int64_t n_frames, void* d_out,
               int64_t o_plane, void* stream);
int wts_power(const float* d_y, int64_t ldy, int64_t n_frames, void* d_out, int64_t ldo, int64_t o_plane,
              void* stream);
int wts_logmel_max(const float* d_m, int64_t n, float* d_max, void* stream);
int wts_logmel_finish(const float* d_m, int64_t n_frames, int32_t n_mels, const float* d_max, float* d_out_f32,
                      void* stream);

/* Gathers 30-s windows of the log-mel (zero padded past `segment_size`, like pad_or_trim) into the padded
 * conv1 input [B, 3002, n_mels] SB16.  d_mel_ptr[b]: device address of window b's time-major float32 log-mel
 * [frames, n_mels]; d_seek[b] / d_size[b]: first frame and number of content frames of the window. */
int wts_window_gather(const int64_t* d_mel_ptr, int32_t n_mels, const int32_t* d_seek, const int32_t* d_size,
                      int32_t B, void* d_out, int64_t o_plane, void* stream);

/* Decoder token embedding + learned positions for a ragged token batch: row r <- emb[token[r]] + pos[position[r]]. */
int wts_embed(const int32_t* d_tokens, const int32_t* d_positions, const float* d_emb, const float* d_pos,
              int32_t rows, int32_t D, float* d_out, void* stream);

/* out[r] = x[idx[r]] (float32 rows). */
int wts_gather_rows(const float* d_x, int64_t ldx, const int32_t* d_idx, int32_t rows, int32_t D, float* d_out,
                    void* stream);

/* Decoder attention for a ragged token batch (one query row per (sequence, position)).
 * kind 0: causal self-attention over the sequence's KV cache (keys 0..position);
 * kind 2: the same for a decode step (ONE row per sequence): d_q points at packed [q | k | v] rows (ldq = 3*D) and
 *         every (row, head) CTA first appends its K/V of the new position to the cache — wts_kv_append fused in;
 * kind 1: cross-attention over the 1500 encoder positions; when d_qk_out != NULL the PRE-softmax
 *         scores of head `h` are written to d_qk_out[(seq*N + slot)*qk_rows + qk_row[r]] for every head
 *         whose d_head_slot[h] >= 0 (= the alignment heads; replaces hook_attention_weights T.py:783-793).
 * q: float32 [rows, D] (ldq); K/V caches float32 head-major [seq][H][ctx][64].
 * d_row_active (may be NULL): rows with 0 are skipped (finished sequences stop streaming their K/V). */
int wts_decoder_attention(int32_t kind, const float* d_q, int64_t ldq, const float* d_k, const float* d_v,
                          int64_t seq_stride, int32_t ctx, const int32_t* d_row_seq, const int32_t* d_row_pos,
                          int32_t rows, int32_t H, void* d_out_sb16, int64_t ldo, int64_t o_plane,
                          float* d_qk_out, const int32_t* d_head_slot, int32_t n_slots, int32_t qk_rows,
                          const int32_t* d_qk_row, const int32_t* d_row_active, void* stream);

/* Cross-attention with fp16 K/V caches (decode-time cross-attention is an HBM stream of K/V; fp16 halves
 * it).  The alignment heads (d_head_slot[h] >= 0) read a float32 copy of K so the exported pre-softmax rows
 * stay within 1e-3 of the reference; see csrc/ops.cu.
 * wts_cross_kv_pack: float32 head-major [B][H][ctx][64] -> fp16 cache (+ float32 [B][n_slots][ctx][64] copy of
 *                    the alignment heads when d_dst_align != NULL). */
int wts_cross_kv_pack(const float* d_src, void* d_dst16, float* d_dst_align, const int32_t* d_head_slot,
                      int32_t n_slots, int32_t B, int32_t H, int32_t ctx, void* stream);
int wts_cross_attention_f16(const float* d_q, int64_t ldq, const void* d_k16, const void* d_v16,
                            const float* d_k_align, const int32_t* d_head_slot, int32_t n_slots, int32_t ctx,
                            const int32_t* d_row_seq, int32_t rows, int32_t H, void* d_out_sb16, int64_t ldo,
                            int64_t o_plane, float* d_qk_out, int32_t qk_rows, const int32_t* d_qk_row,
                            const int32_t* d_row_active, void* stream);
/* Per-layer compacted float32 K copy.  The slots of the alignment heads are numbered layer-major, so the heads of one
 * decoder layer hold the contiguous slots [align_s0, align_s0 + align_n) and the layer's float32 K copy is
 * [B][align_n][ctx][64]: head h of window b sits at (b * align_n + head_slot[h] - align_s0).  The alignment buffer
 * d_qk_out keeps every slot: [B][n_slots][qk_rows][ctx].  A layer without alignment heads passes align_n = 0 and no
 * copy.  wts_cross_kv_pack / wts_cross_attention_f16 are these entries with align_s0 = 0, align_n = n_slots. */
int wts_cross_kv_pack_layer(const float* d_src, void* d_dst16, float* d_dst_align, const int32_t* d_head_slot,
                            int32_t align_s0, int32_t align_n, int32_t B, int32_t H, int32_t ctx, void* stream);
int wts_cross_attention_f16_layer(const float* d_q, int64_t ldq, const void* d_k16, const void* d_v16,
                                  const float* d_k_align, const int32_t* d_head_slot, int32_t n_slots, int32_t align_s0,
                                  int32_t align_n, int32_t ctx, const int32_t* d_row_seq, int32_t rows, int32_t H,
                                  void* d_out_sb16, int64_t ldo, int64_t o_plane, float* d_qk_out, int32_t qk_rows,
                                  const int32_t* d_qk_row, const int32_t* d_row_active, void* stream);

/* Scatter new self-attention K/V rows (float32 [rows, D]) into the head-major caches at (seq, position). */
int wts_kv_append(const float* d_k, const float* d_v, int64_t ld, const int32_t* d_row_seq,
                  const int32_t* d_row_pos, int32_t rows, int32_t H, int32_t ctx, float* d_kc, float* d_vc,
                  int64_t seq_stride, void* stream);

/* Logit filters + greedy choice for one decode step — replaces SuppressBlank / SuppressTokens /
 * ApplyTimestampRules / GreedyDecoder.update (upstream whisper.decoding; rebuilt by the reference at
 * T.py:1371-1393 and re-applied in hook_output_logits T.py:871-875).  One CTA per sequence.
 * d_full_logprobs (optional, [B, lp_ld, V]): every filtered log-softmax row (tests).  d_last_full (optional, [B, V]):
 * the filtered log-softmax row of the step that reaches the decoding limit — the reference reads
 * chunk_logprobs[-1][fallback token] there (T.py:529-538, 735). */
typedef struct WtsDecodeCfg {
    int32_t n_vocab, eot, timestamp_begin, no_timestamps, max_initial_ts;   /* max_initial_ts < 0: none */
    int32_t sample_len, n_ctx, tokens_ld;
} WtsDecodeCfg;
int wts_decode_select(float* d_logits, int64_t ldl, const WtsDecodeCfg* cfg, const uint8_t* d_suppress,
                      const uint8_t* d_blank, int32_t* d_tokens, int32_t* d_n_tokens, const int32_t* d_n_prompt,
                      int32_t* d_done, float* d_logprobs, int32_t lp_ld, float* d_full_logprobs,
                      float* d_last_full, int32_t B, void* stream);

/* The filtered log-softmax row of every sequence (same filters as wts_decode_select, no choice and no state update):
 * what upstream's BeamSearchDecoder.update / GreedyDecoder.update (temperature > 0) consume.  d_out: [B, V]. */
int wts_filtered_logprobs(const float* d_logits, int64_t ldl, const WtsDecodeCfg* cfg, const uint8_t* d_suppress,
                          const uint8_t* d_blank, int32_t* d_tokens, int32_t* d_n_tokens, const int32_t* d_n_prompt,
                          float* d_out, int32_t B, void* stream);

/* ---- Decoder step for small active batches (csrc/decode_steps.cu).
 * One whole decoder step (embed, all blocks with KV-cache append, causal self-attention, fp16 cross-attention with the
 * alignment heads' pre-softmax rows written into qk_buf, final LayerNorm, tied-embedding logits, logit filters +
 * log-softmax + greedy choice) for the sequences whose done flag is 0 — at most 32.  Replaces upstream
 * DecodingTask._main_loop driven through the reference's hooks (T.py:783-793, 849-881), for the whole batch at once.
 * Matrix weights are SB16 planes; q/k projections carry the d_head^-1/4 scale; the self K/V caches, cross K/V caches,
 * token buffers, log-prob rows and qk_buf are the SAME buffers the per-operator path uses, so the two paths can
 * alternate between steps. */
typedef struct WtsDecLayer {
    const float *ln1_g, *ln1_b, *b_qkv, *b_o;                        /* self-attention block */
    const float *ln2_g, *ln2_b, *b_cq, *b_co;                        /* cross-attention block (K/V are cached) */
    const float *ln3_g, *ln3_b, *b_fc1, *b_fc2;                      /* MLP */
    float *self_k, *self_v;                                          /* [cap, H, n_ctx, 64] float32 */
    const void *cross_k16, *cross_v16;                               /* [cap, H, n_audio_ctx, 64] fp16 */
    const float* cross_k_align;                                      /* [cap, align_n, n_audio_ctx, 64] float32 */
    const int32_t* head_slot;                                        /* [H]: alignment slot of each head or -1 */
    /* the six matrices as split-bf16 (SB16) planes [2][out][in] (hi plane at the pointer, lo plane `pl_*` ELEMENTS
     * further), row pitch = in */
    const void *sb_qkv, *sb_o, *sb_cq, *sb_co, *sb_fc1, *sb_fc2;
    int64_t pl_qkv, pl_o, pl_cq, pl_co, pl_fc1, pl_fc2;
    int32_t align_s0, align_n;                                       /* this layer's slots [align_s0, align_s0 + align_n) */
} WtsDecLayer;

typedef struct WtsDecodeSteps {
    const WtsDecLayer* layers;                                       /* device array [n_layer] */
    const float *emb, *pos, *ln_g, *ln_b;                            /* [V, D] float32 (embedding rows), [n_ctx, D], final LayerNorm */
    int32_t *tokens, *n_tokens;
    const int32_t* n_prompt;
    int32_t* done;
    float *logprobs, *full, *last_full, *qk_buf;                     /* full / last_full optional */
    const uint8_t *suppress, *blank;
    float *x, *qkv, *att, *q, *mid, *logits;                         /* scratch: [cap, D], [cap, 3D], [cap, D], [cap, D], [cap, 4D], [cap, V] */
    const void* emb_sb;                                              /* token embedding as SB16 planes (logits) */
    int64_t emb_plane;
    WtsDecodeCfg cfg;
    int32_t n_layer, D, H, n_ctx, n_audio_ctx, n_slots, cap, lp_ld, qk_rows, max_rows;
} WtsDecodeSteps;

/* One step as a chain of per-phase kernels under programmatic dependent launch (2 + 8 n_layer + 1 launches; meant to
 * be captured in a CUDA graph and replayed once per token): each kernel pulls its weight rows into L2 while its
 * producer drains.  h_layers: HOST copy of the layer table p->layers points to.  p->max_rows (1..32) sizes the grids.
 * Returns < 0 with a message for unsupported dimensions, or when the device has fewer than D / 16 SMs. */
int wts_decode_step_kernels(const WtsDecodeSteps* p, const WtsDecLayer* h_layers, void* stream);

/* Per-step decoder inputs from the token buffers: tok[b] = last token, pos[b] = its position,
 * qk_row[b] = number of tokens sampled so far (row that the step predicts), or -1 when the sequence is done. */
int wts_step_inputs(const int32_t* d_tokens, int32_t tokens_ld, const int32_t* d_n_tokens, const int32_t* d_n_prompt,
                    const int32_t* d_done, int32_t B, int32_t* d_tok, int32_t* d_pos, int32_t* d_qk_row,
                    int32_t* d_active, void* stream);

/* probability of <|nospeech|> at the <|startoftranscript|> position (T.py:856-859). */
int wts_softmax_pick(const float* d_logits, int64_t ldl, int32_t n, int32_t index, float* d_out, int32_t rows,
                     void* stream);

/* d_out[i] = log_softmax(d_logits[d_rows[i]])[d_tokens[i]]: teacher-forced token log-probabilities of the two-pass
 * strategy (F.log_softmax + gather, T.py:1245-1246, 1285-1300). */
int wts_logprob_gather(const float* d_logits, int64_t ldl, int32_t n, const int32_t* d_rows, const int32_t* d_tokens,
                       float* d_out, int32_t count, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* WTS_H */
