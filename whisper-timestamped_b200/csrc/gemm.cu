// GEMM of libwts: C = act(alpha * A * B^T + bias) + residual on split-bf16 ("SB16") operands.
//   backend 1: SIMT float32 kernel (validator / small problems / float32-operand log-mel GEMMs)
//   backend 0: wgmma tensor-core kernel (gemm_tc.cu)
#include <cuda_bf16.h>

#include "common.cuh"

namespace wts {

int gemm_tc_launch(const WtsGemm& g, cudaStream_t st);   // gemm_tc.cu

__device__ __forceinline__ float ld_operand(const void* p, int64_t idx, int64_t plane, bool is_f32)
{
    if (is_f32) return reinterpret_cast<const float*>(p)[idx];
    const __nv_bfloat16* q = reinterpret_cast<const __nv_bfloat16*>(p);
    return __bfloat162float(q[idx]) + __bfloat162float(q[idx + plane]);
}

__device__ __forceinline__ float gelu_erf(float v) { return 0.5f * v * (1.0f + erff(v * 0.70710678118654752440f)); }

__device__ __forceinline__ void gemm_epilogue_store(const WtsGemm& g, int zo, int zi, int m, int n, float acc)
{
    float v = g.alpha * acc;
    if (g.bias) v += g.bias[g.bias_on_m ? m : n];
    if (g.act == 1) v = gelu_erf(v);
    if (g.residual) v += g.residual[(int64_t)zo * g.r_bo + (int64_t)zi * g.r_bi + (int64_t)m * g.ldr + n];
    if (g.out_f32) {
        const int64_t off = g.head_dim > 0 ? (int64_t)(n / g.head_dim) * g.head_stride + (int64_t)m * g.ldc + (n % g.head_dim)
                                           : (int64_t)m * g.ldc + n;
        g.out_f32[(int64_t)zo * g.c_bo + (int64_t)zi * g.c_bi + off] = v;
    }
    if (g.out_sb16) {
        const int64_t off = g.head_dim > 0 ? (int64_t)(n / g.head_dim) * g.head_stride + (int64_t)m * g.ldo + (n % g.head_dim)
                                           : (int64_t)m * g.ldo + n;
        __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(g.out_sb16) + (int64_t)zo * g.o_bo + (int64_t)zi * g.o_bi + off;
        const __nv_bfloat16 hi = __float2bfloat16_rn(v);
        o[0] = hi;
        o[g.o_plane] = __float2bfloat16_rn(v - __bfloat162float(hi));
    }
}

constexpr int ST = 64, SK = 16;
__global__ void __launch_bounds__(256)
gemm_simt_kernel(const WtsGemm g)
{
    __shared__ float As[SK][ST + 4];
    __shared__ float Bs[SK][ST + 4];
    const int z = blockIdx.z, zo = z / g.batch_inner, zi = z % g.batch_inner;
    const int m0 = blockIdx.y * ST, n0 = blockIdx.x * ST;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int64_t abase = (int64_t)zo * g.a_bo + (int64_t)zi * g.a_bi;
    const int64_t bbase = (int64_t)zo * g.b_bo + (int64_t)zi * g.b_bi;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < g.K; k0 += SK) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int e = threadIdx.x + i * 256;          // 0..1023
            const int r = e >> 4, kk = e & 15;
            const int m = m0 + r, n = n0 + r, k = k0 + kk;
            As[kk][r] = (m < g.M && k < g.K) ? ld_operand(g.a, abase + (int64_t)m * g.lda + k, g.a_plane, g.a_is_f32) : 0.f;
            Bs[kk][r] = (n < g.N && k < g.K) ? ld_operand(g.b, bbase + (int64_t)n * g.ldb + k, g.b_plane, g.b_is_f32) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < SK; ++kk) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
            if (m < g.M && n < g.N) gemm_epilogue_store(g, zo, zi, m, n, acc[i][j]);
        }
}

}  // namespace wts

using namespace wts;

extern "C" int wts_gemm(const WtsGemm* gp, void* stream)
{
    if (!gp) { set_error("wts_gemm: null descriptor"); return -2; }
    const WtsGemm g = *gp;
    if (g.M <= 0 || g.N <= 0 || g.batch_outer <= 0 || g.batch_inner <= 0) return 0;
    if (!g.a || !g.b || (!g.out_f32 && !g.out_sb16)) { set_error("wts_gemm: null operand/output"); return -2; }
    cudaStream_t st = (cudaStream_t)stream;
    if (g.backend == 0 && !g.a_is_f32 && !g.b_is_f32) return gemm_tc_launch(g, st);
    dim3 grid((g.N + ST - 1) / ST, (g.M + ST - 1) / ST, g.batch_outer * g.batch_inner);
    gemm_simt_kernel<<<grid, 256, 0, st>>>(g);
    WTS_LAUNCH_CHECK();
    return 0;
}
