// ridge.cuh — the ridge regression of Pearl's LinearRegression (neural_networks/contextual_bandit/linear_regression.py)
// shared by the learners that fit one on feature rows: LinearBandit (bandit.cu, rows = state || action features) and
// NeuralLinearBandit (neural_linear.cu, rows = the network's output).  The row load, the fixed-order statistics and their
// reduction into A, b and sum_weight, the discounting decision with the fp64 Gauss-Jordan solve, and the first-maximum
// argmax of the UCB scores.  bandit.cu's header describes the numerics.  The row load, the scoring feature rows
// (k_cb_feat) and the argmax also serve NeuralBandit (neural_bandit.cu), which has no ridge.  The statistics, reduction,
// solve, sampler and score-row bodies are __device__ functions that the one-ridge kernels here and the per-arm kernels
// of the disjoint learners (disjoint_bandit.cu) both call.
//
// Every kernel is `static`: each translation unit that includes this header has its own copy, so the solve's dynamic
// shared-memory attribute is set per unit (cb_solve_prepare, called from each learner's create).
#pragma once
#include <math.h>

#include "common.cuh"
#include "rounds.cuh"

namespace prl {

constexpr int kMaxD = 128;     // ridge width + 1 (the intercept): d^2 doubles fill 128 KB of shared memory
constexpr int kChunk = 256;    // rows per partial sum of k_cb_stats
constexpr int kStage = 32;     // rows staged in shared memory at a time
constexpr int kSolveThreads = 512;

// entries of one partial: the packed lower triangle of x^T (x w) (row i, column j <= i at i (i + 1) / 2 + j), then the d
// entries of x^T (y w), then sum w
__host__ __device__ inline int cb_entries(int d) { return d * (d + 1) / 2 + d + 1; }

// rows of one round: X[b] = state || action features, Y[b], W[b].  records == null: the caller's dense batch.  Call: the
// learner's per-call block, with `slots` and the dense-batch fields d_state, d_action, d_action_ld, d_reward, d_weight.
// rep 1: one-hot of the stored id over act_dim columns; rep 2: its act_dim low bits (bit p at column p)
template <class Call>
static __global__ void k_cb_load(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int act_dim, int rep,
                          const Call *__restrict__ call, const int *__restrict__ round_idx, int B, float *__restrict__ X,
                          float *__restrict__ Y, float *__restrict__ W) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    const int k = obs + act_dim;
    float *x = X + (size_t)w * k;
    if (!records) {
        for (int p = lane; p < obs; p += 32) x[p] = call->d_state[(size_t)w * obs + p];
        for (int p = lane; p < act_dim; p += 32) x[obs + p] = call->d_action[(size_t)w * call->d_action_ld + p];
        if (lane == 0) {
            Y[w] = call->d_reward[w];
            W[w] = call->d_weight ? call->d_weight[w] : 1.f;
        }
        return;
    }
    const int32_t *slots = call->slots + (size_t)(*round_idx) * B;
    const uint32_t *r = records + (size_t)slots[w] * L.record_words;
    for (int p = lane; p < obs; p += 32) x[p] = __uint_as_float(r[L.off_state + p]);
    const int id = (int)r[L.off_action];
    for (int p = lane; p < act_dim; p += 32) x[obs + p] = rep == 1 ? (p == id ? 1.f : 0.f) : (((id >> p) & 1) ? 1.f : 0.f);
    if (lane == 0) {
        Y[w] = __uint_as_float(r[L.off_reward]);
        W[w] = 1.f;
    }
}

// feature rows [r0, r0 + m) of the n x S scoring rows: X[i] = state[s] || act_feat[a] (row = s S + a), one warp per row
static __global__ void k_cb_feat(int m, long long r0, int S, int obs, int act_dim, const float *__restrict__ state,
                          const float *__restrict__ act_feat, float *__restrict__ X) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= m) return;
    const long long row = r0 + w;
    const int s = (int)(row / S), a = (int)(row - (long long)s * S), k = obs + act_dim;
    float *x = X + (size_t)w * k;
    for (int p = lane; p < obs; p += 32) x[p] = state[(size_t)s * obs + p];
    for (int p = lane; p < act_dim; p += 32) x[obs + p] = act_feat[(size_t)a * act_dim + p];
}

// partial sums of the rows of chunk c = blockIdx.x - chunk0 (rows [c kChunk, +kChunk) of the B rows) into P[c][e], one
// entry per thread (blockIdx.y selects the entries), rows in ascending order.  The rows [1, x] are staged kStage at a time
// with x w and y w beside them.  The body of k_cb_stats (chunk0 = 0) and of the per-arm k_dj_stats.
static __device__ __forceinline__ void cb_stats_chunk(int B, int k, const float *__restrict__ X, const float *__restrict__ Y,
                                                      const float *__restrict__ W, float *__restrict__ P, unsigned chunk0) {
    __shared__ float xs[kStage][kMaxD], xws[kStage][kMaxD], yw[kStage], ws[kStage];
    const int d = k + 1, T = d * (d + 1) / 2, E = T + d + 1;
    const int e = blockIdx.y * blockDim.x + threadIdx.x;
    // the entry's operands: kind 0 = A[i][j], 1 = b[i], 2 = sum w
    int kind = 2, i = 0, j = 0;
    if (e < T) {
        kind = 0;
        i = (int)((sqrtf(8.f * (float)e + 1.f) - 1.f) * 0.5f);
        while (i * (i + 1) / 2 > e) i--;
        while ((i + 1) * (i + 2) / 2 <= e) i++;
        j = e - i * (i + 1) / 2;
    } else if (e < T + d) {
        kind = 1;
        i = e - T;
    }
    const unsigned chunk = blockIdx.x - chunk0;
    const int r0 = chunk * kChunk, r1 = min(B, r0 + kChunk);
    float acc = 0.f;
    for (int s0 = r0; s0 < r1; s0 += kStage) {
        const int n = min(kStage, r1 - s0);
        __syncthreads();
        for (int t = threadIdx.x; t < n * d; t += blockDim.x) {
            const int rr = t / d, c = t - rr * d;
            const float v = c == 0 ? 1.f : X[(size_t)(s0 + rr) * k + c - 1];
            xs[rr][c] = v;
            xws[rr][c] = __fmul_rn(v, W[s0 + rr]);
        }
        for (int t = threadIdx.x; t < n; t += blockDim.x) {
            yw[t] = __fmul_rn(Y[s0 + t], W[s0 + t]);
            ws[t] = W[s0 + t];
        }
        __syncthreads();
        if (e < E) {
            if (kind == 0)
                for (int rr = 0; rr < n; rr++) acc = fmaf(xs[rr][i], xws[rr][j], acc);
            else if (kind == 1)
                for (int rr = 0; rr < n; rr++) acc = fmaf(xs[rr][i], yw[rr], acc);
            else
                for (int rr = 0; rr < n; rr++) acc = __fadd_rn(acc, ws[rr]);
        }
    }
    if (e < E) P[(size_t)chunk * E + e] = acc;
}

static __global__ void __launch_bounds__(256) k_cb_stats(int B, int k, const float *__restrict__ X, const float *__restrict__ Y,
                                                  const float *__restrict__ W, float *__restrict__ P) {
    cb_stats_chunk(B, k, X, Y, W, P, 0);
}

// entry blockIdx.x blockDim.x + threadIdx.x of the chunks' partials added in ascending chunk order, then added into A (both triangles), b and sum_weight.
// The body of k_cb_reduce and of the per-arm k_dj_reduce.
static __device__ __forceinline__ void cb_reduce_entry(int d, int chunks, const float *__restrict__ P, float *__restrict__ A,
                                                       float *__restrict__ b, float *__restrict__ sum_weight) {
    const int T = d * (d + 1) / 2, E = T + d + 1;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= E) return;
    float s = 0.f;
    for (int c = 0; c < chunks; c++) s = __fadd_rn(s, P[(size_t)c * E + e]);
    if (e < T) {
        int i = (int)((sqrtf(8.f * (float)e + 1.f) - 1.f) * 0.5f);
        while (i * (i + 1) / 2 > e) i--;
        while ((i + 1) * (i + 2) / 2 <= e) i++;
        const int j = e - i * (i + 1) / 2;
        A[(size_t)i * d + j] = __fadd_rn(A[(size_t)i * d + j], s);
        if (i != j) A[(size_t)j * d + i] = __fadd_rn(A[(size_t)j * d + i], s);
    } else if (e < T + d) {
        b[e - T] = __fadd_rn(b[e - T], s);
    } else {
        *sum_weight = __fadd_rn(*sum_weight, s);
    }
}

static __global__ void k_cb_reduce(int d, int chunks, const float *__restrict__ P, float *__restrict__ A, float *__restrict__ b,
                            float *__restrict__ sum_weight) {
    cb_reduce_entry(d, chunks, P, A, b, sum_weight);
}

// _maybe_apply_discounting, then calculate_coefs, by one CTA: M = A + lambda I in fp64 shared memory [d][d], inverted in
// place by Gauss-Jordan elimination with partial pivoting (first largest |pivot|, as LAPACK's idamax picks), the row
// exchanges undone as column exchanges at the end.  The body of k_cb_solve and of the per-arm k_dj_solve.
static __device__ __forceinline__ void cb_solve_ridge(int d, float lam, float gamma, double interval, float *__restrict__ A,
                                                      float *__restrict__ b, const float *__restrict__ sum_weight,
                                                      double *__restrict__ last_discount, float *__restrict__ inv_A,
                                                      float *__restrict__ coefs) {
    extern __shared__ double sm[];
    double *M = sm, *bb = sm + (size_t)d * d;
    __shared__ double f[kMaxD];
    __shared__ int piv[kMaxD];
    __shared__ int disc;
    const int tid = threadIdx.x, nt = blockDim.x, dd = d * d;
    if (tid == 0) {
        const double sw = (double)*sum_weight;
        disc = interval > 0.0 && sw - *last_discount >= interval;
        if (disc) *last_discount = sw;
    }
    __syncthreads();
    if (disc && gamma < 1.f) {                 // apply_discounting: sum_weight is not discounted
        for (int t = tid; t < dd; t += nt) A[t] = __fmul_rn(A[t], gamma);
        for (int t = tid; t < d; t += nt) b[t] = __fmul_rn(b[t], gamma);
        __syncthreads();
    }
    for (int t = tid; t < dd; t += nt) {
        const int i = t / d, j = t - i * d;
        M[t] = (double)(i == j ? __fadd_rn(A[t], lam) : A[t]);
    }
    for (int t = tid; t < d; t += nt) bb[t] = (double)b[t];
    __syncthreads();
    for (int k = 0; k < d; k++) {
        if (tid < 32) {
            double best = -1.0;
            int bi = d;
            for (int i = k + tid; i < d; i += 32) {
                const double v = fabs(M[(size_t)i * d + k]);
                if (v > best) { best = v; bi = i; }
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) {
                const double ov = __shfl_xor_sync(0xffffffffu, best, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
            }
            if (tid == 0) piv[k] = bi < d ? bi : k;     // a column of NaNs has no pivot row: keep row k
        }
        __syncthreads();
        const int p = piv[k];
        if (p != k)
            for (int j = tid; j < d; j += nt) {
                const double t = M[(size_t)k * d + j];
                M[(size_t)k * d + j] = M[(size_t)p * d + j];
                M[(size_t)p * d + j] = t;
            }
        __syncthreads();
        const double pv = M[(size_t)k * d + k];
        __syncthreads();
        for (int t = tid; t < 2 * d; t += nt) {
            if (t < d) M[(size_t)k * d + t] = (t == k ? 1.0 : M[(size_t)k * d + t]) / pv;
            else f[t - d] = t - d == k ? 0.0 : M[(size_t)(t - d) * d + k];
        }
        __syncthreads();
        for (int t = tid; t < dd; t += nt) {
            const int i = t / d, j = t - i * d;
            if (i == k) continue;
            M[t] = fma(-f[i], M[(size_t)k * d + j], j == k ? 0.0 : M[t]);
        }
        __syncthreads();
    }
    for (int k = d - 1; k >= 0; k--) {
        const int p = piv[k];
        if (p != k)
            for (int i = tid; i < d; i += nt) {
                const double t = M[(size_t)i * d + k];
                M[(size_t)i * d + k] = M[(size_t)i * d + p];
                M[(size_t)i * d + p] = t;
            }
        __syncthreads();
    }
    for (int t = tid; t < dd; t += nt) inv_A[t] = (float)M[t];
    for (int i = tid; i < d; i += nt) {
        double c = 0.0;
        for (int j = 0; j < d; j++) c = fma(M[(size_t)i * d + j], bb[j], c);
        coefs[i] = (float)c;
    }
}

// one CTA: cb_solve_ridge, then round_idx advances (k_cb_predict reads the round it finished)
static __global__ void __launch_bounds__(kSolveThreads) k_cb_solve(int d, float lam, float gamma, double interval, float *__restrict__ A,
                                                            float *__restrict__ b, const float *__restrict__ sum_weight,
                                                            double *__restrict__ last_discount, float *__restrict__ inv_A,
                                                            float *__restrict__ coefs, int *__restrict__ round_idx) {
    cb_solve_ridge(d, lam, gamma, interval, A, b, sum_weight, last_discount, inv_A, coefs);
    if (threadIdx.x == 0) *round_idx += 1;
}

// one warp's row x = [1, state s, action features a] of the scores (the warp's slice x of shared memory): mu = x . coefs
// and, with_sigma, q = x^T inv_A x, both summed over the warp
static __device__ __forceinline__ void cb_row_form(int s, int a, int obs, int act_dim, const float *__restrict__ state,
                                            const float *__restrict__ act_feat, const float *__restrict__ inv_A,
                                            const float *__restrict__ coefs, int with_sigma, float *x, int lane, float &mu,
                                            float &q) {
    const int d = obs + act_dim + 1;
    for (int c = lane; c < d; c += 32)
        x[c] = c == 0 ? 1.f : (c <= obs ? state[(size_t)s * obs + c - 1] : act_feat[(size_t)a * act_dim + c - 1 - obs]);
    __syncwarp();
    mu = 0.f; q = 0.f;
    for (int j = lane; j < d; j += 32) {
        mu = fmaf(x[j], coefs[j], mu);
        if (with_sigma) {
            float t = 0.f;
            for (int i = 0; i < d; i++) t = fmaf(x[i], inv_A[(size_t)i * d + j], t);
            q = fmaf(t, x[j], q);
        }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        mu += __shfl_xor_sync(0xffffffffu, mu, o);
        q += __shfl_xor_sync(0xffffffffu, q, o);
    }
}

// first maximum of each state's scores over the positions whose mask is non-zero (every position when mask is null);
// 0 when no position is available
static __global__ void k_cb_argmax(int n, int S, const float *__restrict__ scores, const uint8_t *__restrict__ mask, int32_t *__restrict__ idx) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n) return;
    int bi = -1;
    float best = 0.f;
    for (int a = 0; a < S; a++) {
        if (mask && !mask[(size_t)s * S + a]) continue;
        const float v = scores[(size_t)s * S + a];
        if (bi < 0 || v > best) { best = v; bi = a; }
    }
    idx[s] = bi < 0 ? 0 : bi;
}

// ThompsonSamplingExplorationLinear's MultivariateNormal(loc = coefs, precision_matrix = A + lambda I).sample() for the
// standard normal draws eps[d] the caller made.  One CTA.  M = A + lambda I is formed in fp32 as LinearRegression.A forms
// it, then factored M = U U^T with U upper triangular in fp64 shared memory [d][d] (right-looking, from the last column
// down; torch factors the index-reversed M, which is the same factorisation).  U overwrites M's upper triangle.  Then
// U^T x = eps by forward substitution in one warp, and theta = coefs + x rounded to fp32: x has covariance
// U^-T U^-1 = M^-1.  *status = 0, or 1 when a pivot is not positive (M is not positive definite, a NaN included), and
// theta is then left unwritten: the reference's argument validation raises there.  The body of k_cb_ts_sample and of the
// per-arm k_dj_ts_sample.
static __device__ __forceinline__ void cb_ts_draw(int d, float lam, const float *__restrict__ A, const float *__restrict__ coefs,
                                                  const float *__restrict__ eps, float *__restrict__ theta, int *__restrict__ status) {
    extern __shared__ double sm[];
    double *M = sm, *r = sm + (size_t)d * d;
    const int tid = threadIdx.x, nt = blockDim.x, dd = d * d;
    for (int t = tid; t < dd; t += nt) {
        const int i = t / d, j = t - i * d;
        M[t] = (double)(i == j ? __fadd_rn(A[t], lam) : A[t]);
    }
    for (int t = tid; t < d; t += nt) r[t] = (double)eps[t];
    __syncthreads();
    for (int k = d - 1; k >= 0; k--) {
        const double p = M[(size_t)k * d + k];
        if (!(p > 0.0)) {                      // every thread read the same pivot: the whole CTA leaves
            if (tid == 0) *status = 1;
            return;
        }
        const double u = sqrt(p);
        __syncthreads();
        for (int i = tid; i <= k; i += nt) M[(size_t)i * d + k] = i == k ? u : M[(size_t)i * d + k] / u;
        __syncthreads();
        for (int t = tid; t < k * k; t += nt) {  // the leading block's upper triangle: M[i][j] -= U[i][k] U[j][k]
            const int i = t / k, j = t - i * k;
            if (i <= j) M[(size_t)i * d + j] = fma(-M[(size_t)i * d + k], M[(size_t)j * d + k], M[(size_t)i * d + j]);
        }
        __syncthreads();
    }
    if (tid >= 32) return;
    for (int j = 0; j < d; j++) {              // x_j = r_j / U[j][j], then r_i -= U[j][i] x_j for i > j, in ascending j
        const double x = r[j] / M[(size_t)j * d + j];
        for (int i = j + 1 + tid; i < d; i += 32) r[i] = fma(-M[(size_t)j * d + i], x, r[i]);
        if (tid == 0) theta[j] = (float)((double)coefs[j] + x);
        __syncwarp();
    }
    if (tid == 0) *status = 0;
}

static __global__ void __launch_bounds__(kSolveThreads) k_cb_ts_sample(int d, float lam, const float *__restrict__ A,
                                                                const float *__restrict__ coefs, const float *__restrict__ eps,
                                                                float *__restrict__ theta, int *__restrict__ status) {
    cb_ts_draw(d, lam, A, coefs, eps, theta, status);
}

static size_t cb_solve_smem(int d) { return ((size_t)d * d + d) * sizeof(double); }

// the attribute belongs to the kernel, not to a handle: raise it to what the widest supported d needs, so that a later
// handle of a smaller d cannot lower it under the launches of a live wider one.  The sampler has the same budget.
static cudaError_t cb_solve_prepare() {
    const cudaError_t e = cudaFuncSetAttribute(k_cb_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cb_solve_smem(kMaxD));
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(k_cb_ts_sample, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cb_solve_smem(kMaxD));
}

// the sampler on `st`, for the learners' ridge buffers
static cudaError_t cb_ts_sample(int d, float lam, const float *A, const float *coefs, const float *eps, float *theta, int *status,
                                cudaStream_t st) {
    k_cb_ts_sample<<<1, kSolveThreads, cb_solve_smem(d), st>>>(d, lam, A, coefs, eps, theta, status);
    return cudaGetLastError();
}

}  // namespace prl
