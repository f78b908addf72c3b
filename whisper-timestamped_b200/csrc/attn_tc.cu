// Fused encoder self-attention on wgmma (sm_90a): softmax(Q K^T) V for 1500 x 1500 positions, head dim 64,
// without ever writing the score matrix to HBM.  Replaces the upstream MultiHeadAttention.qkv_attention of the
// AudioEncoder blocks (reached by the reference through model.transcribe, T.py:904).
//
// One CTA per (128-query tile, head, window); 288 threads:
//   warp 8 (one lane)  TMA producer: the Q tile once, then one 128-key K tile per step (pass 1) or one K tile and the
//                      matching V^T tile (pass 2) into a 2-stage ring
//   warpgroups 0, 1    queries 64*wg .. 64*wg+63: S = Q K^T (bf16x3, wgmma.m64n128k16, both operands in shared memory)
//                      into registers; softmax on the accumulator fragment; O += P V (bf16x3, wgmma.m64n64k16) with the
//                      probabilities as the REGISTER A operand (hi/lo bf16 split of the S fragment, no shared memory)
// Two passes over the keys instead of an online-softmax rescale: pass 1 finds the exact row maxima (S only),
// pass 2 recomputes S, accumulates exp(s - max) and P V, and the epilogue divides by the row sum.  The extra
// Q K^T costs 1/3 more tensor work but no rescaling of O, and the score tile never leaves the SM.
// Operands are SB16 (hi/lo bf16 planes); scale is folded into the q/k projection weights.
#include <cuda_bf16.h>

#include "sm90.cuh"

namespace wts {

constexpr int AT_THREADS = 288;
constexpr int AT_Q = 0, AT_K = 32768, AT_V = 98304, AT_BAR = 163840;
constexpr int AT_SMEM = AT_BAR + 256 + 1024;
// barrier slots (8 bytes each) relative to AT_BAR
enum { B_QFULL = 0, B_FULL = 1, B_EMPTY = 3 };

__device__ __forceinline__ float at_ex2(float x)
{
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

struct AttnArgs {
    __nv_bfloat16* out;      // SB16 [B*n_ctx, ldo]
    int64_t ldo, o_plane;
    int n_ctx, D, H, n_kt;   // n_kt = key tiles of 128
};

// S[64 x 128] of this warpgroup's queries against key tile st of the ring (bf16x3)
__device__ __forceinline__ void scores(float (&s)[64], uint64_t q_hi, uint64_t q_lo, uint32_t k_tile)
{
    const uint64_t k_hi = wg_desc(k_tile), k_lo = wg_desc(k_tile + 16384);
    wg_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint64_t adv = (uint64_t)(2 * k);
        wgmma_ss_n128(s, q_hi + adv, k_hi + adv, k ? 1 : 0);
        wgmma_ss_n128(s, q_lo + adv, k_hi + adv, 1);
        wgmma_ss_n128(s, q_hi + adv, k_lo + adv, 1);
    }
    wg_commit();
    wg_wait<0>();
}

__global__ void __launch_bounds__(AT_THREADS, 1)
enc_attention_tc_kernel(const __grid_constant__ CUtensorMap tmQK, const __grid_constant__ CUtensorMap tmV, const AttnArgs a)
{
    extern __shared__ unsigned char smem_raw[];
    const uint32_t base = (smem_addr(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar = base + AT_BAR;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int q0 = qt * 128;
    const int NT = a.n_kt;

    if (threadIdx.x == 256) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmQK) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmV) : "memory");
        mbar_init(bar + 8 * B_QFULL, 1);
        for (int s = 0; s < 2; ++s) {
            mbar_init(bar + 8 * (B_FULL + s), 1);
            mbar_init(bar + 8 * (B_EMPTY + s), 8);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            // Q tile: columns h*64.., rows q0.. of window b
            mbar_expect_tx(bar + 8 * B_QFULL, 32768);
            tma_load_4d(base + AT_Q, &tmQK, bar + 8 * B_QFULL, h * 64, q0, b, 0);
            tma_load_4d(base + AT_Q + 16384, &tmQK, bar + 8 * B_QFULL, h * 64, q0, b, 1);
            for (int i = 0; i < 2 * NT; ++i) {
                const int j = i % NT, st = i & 1, u = i >> 1;
                const bool pass2 = i >= NT;
                mbar_wait(bar + 8 * (B_EMPTY + st), (u & 1) ^ 1);
                const uint32_t f = bar + 8 * (B_FULL + st);
                mbar_expect_tx(f, pass2 ? 65536 : 32768);
                const uint32_t kt = base + AT_K + st * 32768;
                tma_load_4d(kt, &tmQK, f, a.D + h * 64, j * 128, b, 0);
                tma_load_4d(kt + 16384, &tmQK, f, a.D + h * 64, j * 128, b, 1);
                if (pass2) {
                    // V^T tile: rows h*64.. (channels), columns = keys; two 64-key boxes per plane
                    const uint32_t vt = base + AT_V + st * 32768;
                    tma_load_4d(vt, &tmV, f, j * 128, h * 64, b, 0);
                    tma_load_4d(vt + 8192, &tmV, f, j * 128 + 64, h * 64, b, 0);
                    tma_load_4d(vt + 16384, &tmV, f, j * 128, h * 64, b, 1);
                    tma_load_4d(vt + 24576, &tmV, f, j * 128 + 64, h * 64, b, 1);
                }
            }
        }
        return;
    }

    const int wg = warp >> 2;
    const int cl = 2 * (lane & 3);                  // key / channel column of fragment element 4j: cl + 8j
    const uint64_t q_hi = wg_desc(base + AT_Q + wg * 8192), q_lo = wg_desc(base + AT_Q + 16384 + wg * 8192);
    mbar_wait(bar + 8 * B_QFULL, 0);
    float s[64];
#pragma unroll
    for (int e = 0; e < 64; ++e) s[e] = 0.f;
    // rows r0 = 16*(warp%4) + lane/4 and r0 + 8 of this warpgroup's 64 queries: fragment elements 4j + 0/1 and 4j + 2/3
    float mx[2] = {-INFINITY, -INFINITY};
    for (int i = 0; i < NT; ++i) {                  // pass 1: exact row maxima
        const int st = i & 1, u = i >> 1;
        mbar_wait(bar + 8 * (B_FULL + st), u & 1);
        scores(s, q_hi, q_lo, base + AT_K + st * 32768);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar + 8 * (B_EMPTY + st));
        const int key0 = i * 128 + cl;
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e)
                if (key0 + 8 * j + (e & 1) < a.n_ctx) mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * j + e]);
    }
    float ml2[2], sum[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(FULL_MASK, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(FULL_MASK, mx[r], 2));
        ml2[r] = mx[r] * 1.4426950408889634f;
    }
    float o[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) o[e] = 0.f;
    for (int jt = 0; jt < NT; ++jt) {               // pass 2: probabilities in registers, partial row sums, O += P V
        const int i = NT + jt, st = i & 1, u = i >> 1;
        mbar_wait(bar + 8 * (B_FULL + st), u & 1);
        scores(s, q_hi, q_lo, base + AT_K + st * 32768);
        const int key0 = jt * 128 + cl;
        const bool tail = jt * 128 + 128 > a.n_ctx;
        uint32_t ph[32], pl[32];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                float p0 = at_ex2(fmaf(s[4 * j + 2 * r], 1.4426950408889634f, -ml2[r]));
                float p1 = at_ex2(fmaf(s[4 * j + 2 * r + 1], 1.4426950408889634f, -ml2[r]));
                if (tail) {
                    if (key0 + 8 * j >= a.n_ctx) p0 = 0.f;
                    if (key0 + 8 * j + 1 >= a.n_ctx) p1 = 0.f;
                }
                sum[r] += p0 + p1;
                const __nv_bfloat162 hb = __floats2bfloat162_rn(p0, p1);
                const __nv_bfloat162 lb = __floats2bfloat162_rn(p0 - __low2float(hb), p1 - __high2float(hb));
                // A fragment of k-step j/2: a0 = (r0, keys 0-7), a1 = (r0+8, keys 0-7), a2 / a3 = the same for keys 8-15
                const int idx = 4 * (j >> 1) + 2 * (j & 1) + r;
                ph[idx] = *reinterpret_cast<const uint32_t*>(&hb);
                pl[idx] = *reinterpret_cast<const uint32_t*>(&lb);
            }
        }
        const uint32_t vt = base + AT_V + st * 32768;
        wg_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
            const uint32_t box = vt + (kk >> 2) * 8192;
            const uint64_t v_hi = wg_desc(box) + (uint64_t)(2 * (kk & 3)), v_lo = wg_desc(box + 16384) + (uint64_t)(2 * (kk & 3));
            wgmma_rs_n64(o, ph + 4 * kk, v_hi);
            wgmma_rs_n64(o, pl + 4 * kk, v_hi);
            wgmma_rs_n64(o, ph + 4 * kk, v_lo);
        }
        wg_commit();
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(bar + 8 * (B_EMPTY + st));
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        sum[r] += __shfl_xor_sync(FULL_MASK, sum[r], 1);
        sum[r] += __shfl_xor_sync(FULL_MASK, sum[r], 2);
        const float inv = 1.0f / sum[r];
        const int row = q0 + 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * r;
        if (row >= a.n_ctx) continue;
        __nv_bfloat16* dh = a.out + ((int64_t)b * a.n_ctx + row) * a.ldo + h * 64 + cl;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float y0 = o[4 * j + 2 * r] * inv, y1 = o[4 * j + 2 * r + 1] * inv;
            const __nv_bfloat162 hb = __floats2bfloat162_rn(y0, y1);
            const __nv_bfloat162 lb = __floats2bfloat162_rn(y0 - __low2float(hb), y1 - __high2float(hb));
            *reinterpret_cast<__nv_bfloat162*>(dh + 8 * j) = hb;
            *reinterpret_cast<__nv_bfloat162*>(dh + a.o_plane + 8 * j) = lb;
        }
    }
}

// 4-D bf16 map: (cols, rows, batch, plane)
static int at_make_map(CUtensorMap* tm, const void* ptr, int64_t cols, int64_t rows, int64_t ld, int64_t batch,
                       int64_t batch_stride, int64_t plane, int box_cols, int box_rows, const char* which)
{
    auto enc = tensor_map_encoder();
    if (!enc) { set_error("wts_enc_attention: cuTensorMapEncodeTiled entry point not available"); return -4; }
    if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (ld & 7) || (plane & 7) || (batch_stride & 7)) {
        set_error("wts_enc_attention: operand %s not 16-byte aligned", which);
        return -5;
    }
    cuuint64_t dims[4] = {(cuuint64_t)cols, (cuuint64_t)rows, (cuuint64_t)batch, 2};
    cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)batch_stride * 2, (cuuint64_t)plane * 2};
    cuuint32_t box[4] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows, 1, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("wts_enc_attention: cuTensorMapEncodeTiled(%s) failed with %d", which, (int)r); return -6; }
    return 0;
}

}  // namespace wts

using namespace wts;

extern "C" int wts_enc_attention(const void* d_qk, int64_t ld_qk, int64_t qk_plane, const void* d_vt, int64_t ld_vt,
                                 int64_t vt_plane, int32_t B, int32_t H, int32_t D, int32_t n_ctx, void* d_out,
                                 int64_t ldo, int64_t o_plane, void* stream)
{
    if (B <= 0) return 0;
    if (D != H * 64) { set_error("wts_enc_attention: head dim must be 64 (D=%d H=%d)", D, H); return -2; }
    if ((reinterpret_cast<uintptr_t>(d_out) & 3) || (ldo & 1) || (o_plane & 1)) {
        set_error("wts_enc_attention: output not 4-byte aligned");
        return -5;
    }
    static bool attr_set = false;
    if (!attr_set) {
        WTS_CUDA_CHECK(cudaFuncSetAttribute(enc_attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, AT_SMEM));
        attr_set = true;
    }
    alignas(64) CUtensorMap tmQK, tmV;
    // q|k: [B*n_ctx rows, 2D cols]; per-window row extent n_ctx so tiles never read the next window
    int rc = at_make_map(&tmQK, d_qk, 2 * (int64_t)D, n_ctx, ld_qk, B, (int64_t)n_ctx * ld_qk, qk_plane, 64, 128, "qk");
    if (rc) return rc;
    // V^T: [B*D rows (channels), n_ctx cols (keys)]
    rc = at_make_map(&tmV, d_vt, n_ctx, D, ld_vt, B, (int64_t)D * ld_vt, vt_plane, 64, 64, "vt");
    if (rc) return rc;
    AttnArgs a;
    a.out = reinterpret_cast<__nv_bfloat16*>(d_out);
    a.ldo = ldo; a.o_plane = o_plane;
    a.n_ctx = n_ctx; a.D = D; a.H = H; a.n_kt = (n_ctx + 127) / 128;
    dim3 grid((n_ctx + 127) / 128, H, B);
    enc_attention_tc_kernel<<<grid, AT_THREADS, AT_SMEM, (cudaStream_t)stream>>>(tmQK, tmV, a);
    WTS_LAUNCH_CHECK();
    return 0;
}
