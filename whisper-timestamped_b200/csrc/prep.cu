// Fused attention post-processing for word alignment (sm_90a).
//
// Replaces, for a whole batch of segments at once, the per-segment CPU sequence of
// /root/reference/whisper_timestamped/transcribe.py:
//   1540  weights[..., start_token:end_token]                (frame slice)
//   1545  stack of the alignment heads                       (already only those N heads in d_qk)
//   1546  scipy.ndimage.median_filter(weights, (1,1,9))      (mode='reflect')
//   1547  softmax over frames
//   1548  mean over heads
//   1549  divide by the L2 norm over the token axis
//   1550  negate (-> float64 in the reference; the values are float32-exact, kept as float32)
//   1561-1565 padding mask, 1568 weights[0,0] = weights.min()
//
// Kernel A (rows): one warp per (segment, token) row; for each head: coalesced load of the F-frame
// slice into shared memory (with a reflected 4-sample halo so the filter loop is branch-free), medians
// of 9 computed two adjacent outputs at a time (they share 8 samples: one pruned 8-sorter + two clamps),
// numerically stable softmax (ex2.approx), accumulate the head mean in shared memory; the N*T*F*4 input
// bytes are read exactly once.
// Kernel B (cols): one CTA per segment; per frame column: L2 norm over tokens, divide, negate,
// padding mask, running minimum; finally cost[0,0] = min.  Reads the [T,F] mean twice (L2-hot).
#include "common.cuh"
#include "median9.h"
#include "peaks.h"

namespace wts {

constexpr int PREP_WARPS = 4;

// One head of one token row, by one warp: slice -> median of 9 -> softmax, added to acc[] (first head: stored).
__device__ __forceinline__ void prep_head_row(const float* __restrict__ src, const int F, const int lane, float* xb,
                                              float* mbuf, float* acc, const bool first)
{
    const int npair = (F + 1) >> 1;
    for (int c = lane; c < F; c += 32) xb[c + 4] = __ldg(src + c);
    __syncwarp();
    if (lane < 4) {                                   // scipy 'reflect' halo (periodic for tiny F)
        xb[3 - lane] = xb[4 + wts_reflect_index(-1 - lane, F)];
        xb[F + 4 + lane] = xb[4 + wts_reflect_index(F + lane, F)];
    }
    if (lane == 4) xb[F + 8] = 0.f;
    __syncwarp();
    float mx = -INFINITY;
    for (int p = lane; p < npair; p += 32) {
        const int c = 2 * p;
        float v[10];
        const float2* x2 = reinterpret_cast<const float2*>(xb + c);
#pragma unroll
        for (int k = 0; k < 5; ++k) { const float2 q = x2[k]; v[2 * k] = q.x; v[2 * k + 1] = q.y; }
        float m0, m1;
        wts_median9_pair(v, &m0, &m1);
        mbuf[c] = m0;
        mx = fmaxf(mx, m0);
        if (c + 1 < F) { mbuf[c + 1] = m1; mx = fmaxf(mx, m1); }
    }
    mx = warp_max(mx);
    float sum = 0.f;
    for (int c = lane; c < F; c += 32) {
        const float e = __expf(mbuf[c] - mx);
        mbuf[c] = e;
        sum += e;
    }
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
    if (first) { for (int c = lane; c < F; c += 32) acc[c] = mbuf[c] * inv; }
    else       { for (int c = lane; c < F; c += 32) acc[c] += mbuf[c] * inv; }
    __syncwarp();
}

__device__ __forceinline__ const float* prep_row_src(const float* qk, const WtsSegDesc& sd, const int t, const int N,
                                                     const int Tmax, const int Fmax)
{
    const int row = (t == sd.T - 1) ? sd.last_row : sd.row0 + t;
    return qk + (((int64_t)sd.window * N) * Tmax + row) * (int64_t)Fmax + sd.f0;
}

// Serial over heads: one warp per (segment, token) row walks all N heads.
__global__ void __launch_bounds__(PREP_WARPS * 32)
prep_rows_kernel(const float* __restrict__ qk, const int N, const int Tmax, const int Fmax,
                 const WtsSegDesc* __restrict__ segs, const int pitch, float* __restrict__ cost)
{
    extern __shared__ float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const WtsSegDesc sd = segs[blockIdx.x];
    const int t = blockIdx.y * PREP_WARPS + warp;
    if (t >= sd.T) return;
    const int F = sd.F;
    float* xb = smem + (size_t)warp * 3 * pitch;     // raw slice with a 4-sample reflected halo: xb[i+4] = x[i]
    float* mbuf = xb + pitch;                        // median-filtered -> exp
    float* acc = mbuf + pitch;                       // sum over heads of the softmax rows

    const float* src0 = prep_row_src(qk, sd, t, N, Tmax, Fmax);
    const int64_t head_stride = (int64_t)Tmax * Fmax;
    for (int n = 0; n < N; ++n) prep_head_row(src0 + n * head_stride, F, lane, xb, mbuf, acc, n == 0);
    const int P = seg_pitch(sd);
    float* dst = cost + sd.cost_off + (int64_t)t * P;
    const float fn = (float)N;
    for (int c = lane; c < P; c += 32) dst[c] = c < F ? acc[c] / fn : 0.f;     // padding columns (pitch) hold zeros
}

// Head-parallel: one CTA per (segment, token) row; warp w takes heads w, w + PREP_WARPS, ... into its own shared row,
// then the CTA adds the warps' rows in warp order (fixed order: the result does not depend on timing).  For the
// many-head sets (every head of the top layers: 100-320 heads), where the serial walk is 10-30x the work per row.
__global__ void __launch_bounds__(PREP_WARPS * 32)
prep_rows_heads_kernel(const float* __restrict__ qk, const int N, const int Tmax, const int Fmax,
                       const WtsSegDesc* __restrict__ segs, const int pitch, float* __restrict__ cost)
{
    extern __shared__ float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const WtsSegDesc sd = segs[blockIdx.x];
    const int t = blockIdx.y;
    if (t >= sd.T) return;                           // whole CTA: no barrier is skipped by part of it
    const int F = sd.F;
    float* xb = smem + (size_t)warp * 3 * pitch;
    float* mbuf = xb + pitch;
    float* acc = mbuf + pitch;
    const float* src0 = prep_row_src(qk, sd, t, N, Tmax, Fmax);
    const int64_t head_stride = (int64_t)Tmax * Fmax;
    for (int n = warp; n < N; n += PREP_WARPS) prep_head_row(src0 + n * head_stride, F, lane, xb, mbuf, acc, n == warp);
    __syncthreads();
    const int nw = min(N, PREP_WARPS);
    const int P = seg_pitch(sd);
    float* dst = cost + sd.cost_off + (int64_t)t * P;
    const float fn = (float)N;
    for (int c = threadIdx.x; c < P; c += blockDim.x) {
        float s = 0.f;
        if (c < F) {
            s = smem[2 * pitch + c];
            for (int w = 1; w < nw; ++w) s += smem[(size_t)w * 3 * pitch + 2 * pitch + c];
            s /= fn;
        }
        dst[c] = s;
    }
}

__global__ void __launch_bounds__(256)
prep_cols_kernel(const WtsSegDesc* __restrict__ segs, float* __restrict__ cost)
{
    __shared__ float red[8];
    const WtsSegDesc sd = segs[blockIdx.x];
    const int T = sd.T, F = sd.F, P = seg_pitch(sd);
    float* M = cost + sd.cost_off;
    const bool masked = sd.max_dur > 0 && sd.f0 < sd.max_dur;
    float vmin = INFINITY;
    for (int c = threadIdx.x; c < F; c += blockDim.x) {
        float ss = 0.f;
        for (int t = 0; t < T; ++t) {
            const float v = M[(int64_t)t * P + c];
            ss += v * v;
        }
        const float nrm = sqrtf(ss);
        for (int t = 0; t < T; ++t) {
            float v = -(M[(int64_t)t * P + c] / nrm);
            if (masked && t < T - 1 && c >= sd.max_dur) v = 0.f;
            M[(int64_t)t * P + c] = v;
            vmin = fminf(vmin, v);
        }
    }
    vmin = warp_min(vmin);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = vmin;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = red[0];
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) m = fminf(m, red[w]);
        M[0] = m;
    }
}

// detect_disfluencies (T.py:1656-1683): for every token row of every segment, the peak analysis of the (negated) cost
// row between the token's two DTW jumps (peaks.h = scipy.signal.find_peaks(width=3, prominence=0.02) restated).
// One thread per (segment, token): the slices are a few dozen frames, the analysis is a handful of short scans.
__global__ void disfluency_kernel(const float* __restrict__ cost, const WtsSegDesc* __restrict__ segs,
                                  const int32_t* __restrict__ jumps, int32_t* __restrict__ out)
{
    const WtsSegDesc sd = segs[blockIdx.x];
    const int32_t* j = jumps + sd.jumps_off;
    int32_t* o = out + sd.jumps_off;
    for (int t = threadIdx.x; t <= sd.T; t += blockDim.x) {
        int left = -1;
        if (t < sd.T) {
            const int begin = j[t], end = j[t + 1];
            if (end - begin >= 3 && begin >= 0 && end <= sd.F)
                left = wts_disfluency_left(cost + sd.cost_off + (int64_t)t * seg_pitch(sd), begin, end - begin, 0.02, 3.0);
        }
        o[t] = left;
    }
}

}  // namespace wts

using namespace wts;

extern "C" int wts_disfluency_starts(const float* d_cost, const WtsSegDesc* d_segs, int32_t nseg, const int32_t* d_jumps,
                                     int32_t* d_out, void* stream)
{
    if (nseg <= 0) return 0;
    if (!d_cost || !d_segs || !d_jumps || !d_out) { set_error("wts_disfluency_starts: null pointer"); return -2; }
    disfluency_kernel<<<nseg, 64, 0, (cudaStream_t)stream>>>(d_cost, d_segs, d_jumps, d_out);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_attn_prep_batch_kernel(const float* d_qk, int32_t N, int32_t Tmax, int32_t Fmax,
                                          const WtsSegDesc* d_segs, int32_t nseg, int32_t max_T, int32_t max_F,
                                          float* d_cost, int32_t kernel, void* stream)
{
    if (nseg <= 0) return 0;
    if (!d_qk || !d_segs || !d_cost) { set_error("wts_attn_prep_batch: null pointer"); return -2; }
    if (N <= 0 || max_T <= 0 || max_F <= 0 || max_F > Fmax) {
        set_error("wts_attn_prep_batch: bad geometry N=%d max_T=%d max_F=%d Fmax=%d", N, max_T, max_F, Fmax);
        return -2;
    }
    if (kernel < 0 || kernel > 2) { set_error("wts_attn_prep_batch_kernel: kernel %d is not 0, 1 or 2", kernel); return -2; }
    if (kernel == 0) kernel = N >= WTS_PREP_HEADS_MIN_N ? 2 : 1;
    cudaStream_t st = (cudaStream_t)stream;
    const int pitch = (max_F + 10 + 1) & ~1;            // halo + even pitch so float2 reads stay aligned
    const size_t smem = (size_t)PREP_WARPS * 3 * pitch * sizeof(float);
    if (kernel == 1) {
        if (smem > 48 * 1024)
            WTS_CUDA_CHECK(cudaFuncSetAttribute(prep_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        dim3 grid(nseg, (max_T + PREP_WARPS - 1) / PREP_WARPS);
        prep_rows_kernel<<<grid, PREP_WARPS * 32, smem, st>>>(d_qk, N, Tmax, Fmax, d_segs, pitch, d_cost);
    } else {
        if (smem > 48 * 1024)
            WTS_CUDA_CHECK(cudaFuncSetAttribute(prep_rows_heads_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        dim3 grid(nseg, max_T);
        prep_rows_heads_kernel<<<grid, PREP_WARPS * 32, smem, st>>>(d_qk, N, Tmax, Fmax, d_segs, pitch, d_cost);
    }
    WTS_LAUNCH_CHECK();
    prep_cols_kernel<<<nseg, 256, 0, st>>>(d_segs, d_cost);
    WTS_LAUNCH_CHECK();
    return 0;
}

extern "C" int wts_attn_prep_batch(const float* d_qk, int32_t N, int32_t Tmax, int32_t Fmax,
                                   const WtsSegDesc* d_segs, int32_t nseg, int32_t max_T,
                                   int32_t max_F, float* d_cost, void* stream)
{
    return wts_attn_prep_batch_kernel(d_qk, N, Tmax, Fmax, d_segs, nseg, max_T, max_F, d_cost, 0, stream);
}
