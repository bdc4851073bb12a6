// umma_test.cu — self-test of the wgmma building block (umma.cuh): one warpgroup computes
// D[M x N] = A[M x K] * B[N x K]^T with plain TF32 or 3xTF32, both operands in shared memory (SS form) or the
// A operand in registers (RS form).  Exposed through the C ABI so tests/ can check it against an fp64 product.
#include <stdarg.h>

#include "common.cuh"
#include "umma.cuh"

using namespace prl;

namespace {

// hi / lo tiles of a row-major [rows x K] matrix with chunk pitch lbo
__device__ void fill_tiles(const float *__restrict__ X, int rows, int K, int lbo, float *hi_t, float *lo_t, bool split) {
    for (int e = threadIdx.x; e < rows * K; e += blockDim.x) {
        const int r = e / K, k = e - r * K;
        const int idx = umma::tile_index2(r, k, K, lbo);
        hi_t[idx] = X[e];
        lo_t[idx] = split ? umma::tf32_lo(X[e]) : 0.f;
    }
}

// rows [row0, row0 + 64) x columns [col0, col0 + N) of D from this warpgroup's accumulator
template <int N>
__device__ __forceinline__ void store_acc(const float *d, float *__restrict__ D, int ldd, int row0, int col0) {
#pragma unroll
    for (int j = 0; j < N / 8; j++)
#pragma unroll
        for (int p = 0; p < 2; p++)
#pragma unroll
            for (int e = 0; e < 2; e++) D[(size_t)(row0 + umma::acc_row(p)) * ldd + col0 + umma::acc_col(j, e)] = d[4 * j + 2 * p + e];
}

template <int N>
__device__ __forceinline__ void block_ss(umma::Tile ah, umma::Tile al, umma::Tile bh, umma::Tile bl, int K, bool plain, float *D,
                                         int ldd, int row0, int col0) {
    float d[N / 2];
    umma::gemm3<N>(d, ah.rows_from(row0), al.rows_from(row0), bh.rows_from(col0), bl.rows_from(col0), K, false, plain, plain);
    umma::wg_commit();
    umma::wg_wait<0>();
    store_acc<N>(d, D, ldd, row0, col0);
}

// SS form: D[M x N] = A[M x K] * B[N x K]^T, M in {64, 128}, N a multiple of 8, operand tiles with chunk pitch `lbo`
// (128 or 144).  plain: one TF32 pass instead of three.
__global__ void __launch_bounds__(128, 1)
k_umma_test_ss(const float *__restrict__ A, const float *__restrict__ B, float *__restrict__ D, int M, int N, int K, int lbo,
               int plain) {
    extern __shared__ __align__(128) float smem[];
    const int a_floats = umma::tile_bytes2(M, K, lbo) / 4, b_floats = umma::tile_bytes2(N, K, lbo) / 4;
    float *a_hi = smem, *a_lo = a_hi + a_floats, *b_hi = a_lo + a_floats, *b_lo = b_hi + b_floats;
    fill_tiles(A, M, K, lbo, a_hi, a_lo, !plain);
    fill_tiles(B, N, K, lbo, b_hi, b_lo, !plain);
    umma::fence_async_smem();
    __syncthreads();
    const umma::Tile ah = umma::make_tile(a_hi, K, lbo), al = umma::make_tile(a_lo, K, lbo);
    const umma::Tile bh = umma::make_tile(b_hi, K, lbo), bl = umma::make_tile(b_lo, K, lbo);
    for (int row0 = 0; row0 < M; row0 += 64) {
        int col0 = 0;
        for (; col0 + 64 <= N; col0 += 64) block_ss<64>(ah, al, bh, bl, K, plain, D, N, row0, col0);
        if ((N - col0) & 32) { block_ss<32>(ah, al, bh, bl, K, plain, D, N, row0, col0); col0 += 32; }
        if ((N - col0) & 16) { block_ss<16>(ah, al, bh, bl, K, plain, D, N, row0, col0); col0 += 16; }
        if ((N - col0) & 8) block_ss<8>(ah, al, bh, bl, K, plain, D, N, row0, col0);
    }
}

template <int N>
__device__ __forceinline__ void block_rs(const float *a_hi, const float *a_lo, umma::Tile bh, umma::Tile bl, int K, float *D, int ldd,
                                         int row0, int col0) {
    float d[N / 2];
    umma::gemm3_rs<N, 8>(d, a_hi, a_lo, bh.rows_from(col0), bl.rows_from(col0), false, K >> 3);
    umma::wg_commit();
    umma::wg_wait<0>();
    store_acc<N>(d, D, ldd, row0, col0);
}

// RS form: every thread loads its own A fragments (hi / lo) from global memory into registers, B in shared memory.
// D[128 x N] = A[128 x K] * B[N x K]^T, K <= 64, N = 32 or a multiple of 64.
__global__ void __launch_bounds__(128, 1)
k_umma_test_rs(const float *__restrict__ A, const float *__restrict__ B, float *__restrict__ D, int N, int K) {
    extern __shared__ __align__(128) float smem[];
    const int b_floats = umma::tile_bytes(N, K) / 4;
    float *b_hi = smem, *b_lo = b_hi + b_floats;
    fill_tiles(B, N, K, 128, b_hi, b_lo, true);
    umma::fence_async_smem();
    __syncthreads();
    const umma::Tile bh = umma::make_tile(b_hi, K, 128), bl = umma::make_tile(b_lo, K, 128);
    const int t = threadIdx.x & 3;
    for (int row0 = 0; row0 < 128; row0 += 64) {
        float hi[32], lo[32];
#pragma unroll
        for (int ks = 0; ks < 8; ks++)
#pragma unroll
            for (int q = 0; q < 2; q++)
#pragma unroll
                for (int p = 0; p < 2; p++) {
                    const int k = 8 * ks + t + 4 * q;
                    const float x = k < K ? A[(size_t)(row0 + umma::acc_row(p)) * K + k] : 0.f;
                    umma::split_tf32(x, hi[4 * ks + 2 * q + p], lo[4 * ks + 2 * q + p]);
                }
        if (N == 32) block_rs<32>(hi, lo, bh, bl, K, D, N, row0, 0);
        else
            for (int col0 = 0; col0 < N; col0 += 64) block_rs<64>(hi, lo, bh, bl, K, D, N, row0, col0);
    }
}

}  // namespace

extern "C" int prl_test_umma_gemm_ts(const float *a_dev, const float *b_dev, float *d_dev, int n, int k, int reps,
                                     void *stream) {
    (void)reps;
    PRL_REQUIRE(a_dev && b_dev && d_dev, "null argument");
    PRL_REQUIRE(n == 32 || (n >= 64 && n <= 256 && n % 64 == 0), "N must be 32 or a multiple of 64 up to 256");
    PRL_REQUIRE(k >= 8 && k % 8 == 0 && k <= 64, "K must be a multiple of 8 in [8,64]");
    const size_t smem = (size_t)2 * umma::tile_bytes(n, k);
    PRL_CUDA(cudaFuncSetAttribute(k_umma_test_rs, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_umma_test_rs<<<1, 128, smem, (cudaStream_t)stream>>>(a_dev, b_dev, d_dev, n, k);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

static int launch_ss(const float *a_dev, const float *b_dev, float *d_dev, int m, int n, int k, int lbo, int plain, void *stream) {
    const size_t smem = (size_t)2 * (umma::tile_bytes2(m, k, lbo) + umma::tile_bytes2(n, k, lbo));
    PRL_REQUIRE(smem <= 200 * 1024, "tile does not fit shared memory");
    PRL_CUDA(cudaFuncSetAttribute(k_umma_test_ss, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_umma_test_ss<<<1, 128, smem, (cudaStream_t)stream>>>(a_dev, b_dev, d_dev, m, n, k, lbo, plain);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

extern "C" int prl_test_umma_gemm2(const float *a_dev, const float *b_dev, float *d_dev, int m, int n, int k,
                                   int lbo, void *stream) {
    PRL_REQUIRE(a_dev && b_dev && d_dev, "null argument");
    PRL_REQUIRE(m == 64 || m == 128, "M must be 64 or 128");
    PRL_REQUIRE(n >= 8 && n <= 256 && n % 8 == 0, "N must be a multiple of 8 in [8,256]");
    PRL_REQUIRE(k >= 8 && k % 8 == 0 && k <= 256, "K must be a multiple of 8 in [8,256]");
    PRL_REQUIRE(lbo >= 128 && lbo % 16 == 0 && lbo <= 512, "lbo must be a multiple of 16 in [128,512]");
    return launch_ss(a_dev, b_dev, d_dev, m, n, k, lbo, 0, stream);
}

extern "C" int prl_test_umma_gemm(const float *a_dev, const float *b_dev, float *d_dev, int n, int k, int passes,
                                  void *stream) {
    PRL_REQUIRE(a_dev && b_dev && d_dev, "null argument");
    PRL_REQUIRE(n >= 16 && n <= 256 && n % 16 == 0 && (n & (n - 1)) == 0, "N must be a power of two in [16,256]");
    PRL_REQUIRE(k >= 8 && k % 8 == 0 && k <= 256, "K must be a multiple of 8 in [8,256]");
    PRL_REQUIRE(passes == 1 || passes == 3, "passes must be 1 or 3");
    return launch_ss(a_dev, b_dev, d_dev, 128, n, k, 128, passes == 1, stream);
}
