// bandit.cu — LinearBandit (LinUCB) driven by PolicyLearner.learn or called directly on a caller's batch
// (PearlAgent.learn_batch / offline_learning), and its UCB scoring, replacing
//   neural_networks/contextual_bandit/linear_regression.py   LinearRegression.learn_batch (A += x^T (x w), symmetrized;
//       b += x^T (y w); sum_weight += sum w), calculate_coefs (inv_A = inv(A + lambda I), coefs = inv_A b),
//       apply_discounting (A, b *= gamma), forward ([1, x] . coefs) and calculate_sigma (sqrt([1, x]^T inv_A [1, x]))
//   policy_learners/contextual_bandits/linear_bandit.py       learn_batch (x = state || represented action, the model's
//       learn_batch, _maybe_apply_discounting, prediction = model(x) after the update), act / get_scores
//   policy_learners/exploration_modules/contextual_bandits/ucb_exploration.py   values + alpha sigma, NaN sigma -> 0
//   policy_learners/exploration_modules/contextual_bandits/thompson_sampling_exploration.py   x . theta with theta from
//       ridge.cuh's k_cb_ts_sample (prl_cb_ts_sample), or with efficient sampling mu + z sigma (k_cb_ts_scores)
//   utils/functional_utils/learning/action_utils.py          get_model_action_index_batch (NO_TIEBREAKING: first max
//       over the available positions)
//
// Round (5 launches, captured once per (batch, buffer) into a CUDA graph and replayed, DESIGN.md §3.4):
//   k_cb_load     the B feature rows x = state || action representation (one-hot or binary code of the stored id, or the
//                 caller's dense action matrix), the label y and the weight w (1, or the caller's vector)
//   k_cb_stats    partial sums of x^T (x w), x^T (y w) and sum w over chunks of kChunk rows, one chunk per CTA column
//   k_cb_reduce   the chunks added in ascending order and added into A, b and sum_weight (fp32, as the reference's buffers)
//   k_cb_solve    one CTA: the discounting decision (in double, as the reference's Python compares .item() floats), then
//                 inv(A + lambda I) by Gauss-Jordan elimination with partial pivoting in fp64 shared memory, rounded to fp32
//                 on the way out, and coefs = inv_A b (fp64, rounded)
//   k_cb_predict  prediction = [1, x] . coefs with the new coefs; label and weight copied out
// No float atomics and a fixed summation order everywhere: bit-reproducible run to run, graph or eager, and independent of
// how the rounds are split into calls.
//
// Why Gauss-Jordan with pivoting rather than Cholesky: like torch.linalg.inv (LU with partial pivoting) it needs no
// positive definiteness, which the fp32 accumulation of A cannot guarantee once A + lambda I is ill-conditioned.
// fp64 keeps the kernel's own rounding far below the fp32 reference's (DESIGN.md, the ridge solve).  With lambda > 0 and
// non-negative weights (the plugin refuses the rest) A + lambda I is nonsingular; non-finite rows (NaN or inf states,
// rewards or weights) propagate into inv_A and coefs as they do through the reference's inverse.
#include <math.h>

#include <new>

#include "common.cuh"
#include "ridge.cuh"
#include "rounds.cuh"

using namespace prl;

namespace {

// per-call block the captured round reads through
struct CbCall {
    const int32_t *slots;                     // [rounds][B] (learn)
    float *out_pred, *out_label, *out_weight; // [rounds][B]
    // learn_batch: the caller's dense batch
    const float *d_state, *d_action, *d_reward, *d_weight;   // d_weight may be null: every weight is 1
    int d_action_ld;                                          // row pitch of d_action (its width)
};

// LinearBandit.learn_batch's report of the round k_cb_solve finished: prediction = model(x) with the new coefs
__global__ void k_cb_predict(int B, int k, const float *__restrict__ X, const float *__restrict__ Y, const float *__restrict__ W,
                             const float *__restrict__ coefs, const CbCall *__restrict__ call, const int *__restrict__ round_idx) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= B) return;
    const size_t o = (size_t)(*round_idx - 1) * B + r;
    const float *x = X + (size_t)r * k;
    float s = coefs[0];
    for (int j = 0; j < k; j++) s = fmaf(x[j], coefs[j + 1], s);
    call->out_pred[o] = s;
    if (call->out_label) call->out_label[o] = Y[r];
    if (call->out_weight) call->out_weight[o] = W[r];
}

// one warp's row x = [1, state s, action features a] of the scores (the warp's slice xw of shared memory): mu = x . coefs
// and, with_sigma, q = x^T inv_A x, both summed over the warp
__device__ __forceinline__ void cb_row_form(int s, int a, int obs, int act_dim, const float *__restrict__ state,
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

// scores of n states x S actions, one warp per (state, action) row x = [1, state, action features a]:
//   mu = x . coefs;  with_sigma: mu + alpha sigma, sigma = sqrt(x^T inv_A x), NaN (a negative form) -> 0
// Thompson sampling scores x . theta through this kernel with coefs = theta and no sigma.
__global__ void __launch_bounds__(256) k_cb_scores(int n, int S, int obs, int act_dim, const float *__restrict__ state,
                                                   const float *__restrict__ act_feat, const float *__restrict__ inv_A,
                                                   const float *__restrict__ coefs, int with_sigma, float alpha,
                                                   float *__restrict__ out) {
    __shared__ float xs[8][kMaxD];
    const int lane = threadIdx.x & 31, wb = threadIdx.x >> 5;
    const long long row = (long long)blockIdx.x * 8 + wb;
    if (row >= (long long)n * S) return;
    const int s = (int)(row / S), a = (int)(row - (long long)s * S);
    float mu, q;
    cb_row_form(s, a, obs, act_dim, state, act_feat, inv_A, coefs, with_sigma, xs[wb], lane, mu, q);
    if (lane == 0) {
        float v = mu;
        if (with_sigma) {
            float sg = sqrtf(q);
            if (isnan(sg)) sg = 0.f;
            v = __fadd_rn(mu, __fmul_rn(alpha, sg));
        }
        out[row] = v;
    }
}

// ThompsonSamplingExplorationLinear with enable_efficient_sampling: torch.normal(mean = mu, std = sigma) for the rows of
// k_cb_scores, given the row's standard normal draw z[row]: z sigma, then + mu, each rounded (no FMA), as torch computes
// it.  A NaN sigma (a negative form) sets *nan_sigma, where torch.normal raises; the UCB path's NaN -> 0 does not apply.
__global__ void __launch_bounds__(256) k_cb_ts_scores(int n, int S, int obs, int act_dim, const float *__restrict__ state,
                                                      const float *__restrict__ act_feat, const float *__restrict__ inv_A,
                                                      const float *__restrict__ coefs, const float *__restrict__ z,
                                                      float *__restrict__ out, int *__restrict__ nan_sigma) {
    __shared__ float xs[8][kMaxD];
    const int lane = threadIdx.x & 31, wb = threadIdx.x >> 5;
    const long long row = (long long)blockIdx.x * 8 + wb;
    if (row >= (long long)n * S) return;
    const int s = (int)(row / S), a = (int)(row - (long long)s * S);
    float mu, q;
    cb_row_form(s, a, obs, act_dim, state, act_feat, inv_A, coefs, 1, xs[wb], lane, mu, q);
    if (lane == 0) {
        const float sg = sqrtf(q);
        if (isnan(sg)) *nan_sigma = 1;
        out[row] = __fadd_rn(mu, __fmul_rn(z[row], sg));
    }
}

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_cb : Rounds<prl_cb, CbCall> {
    static constexpr const char *kFn = "prl_cb", *kName = "LinearBandit";
    prl_cb_cfg cfg;
    int k, d;
    float *A, *b, *sum_weight, *inv_A, *coefs;
    double *last_discount;
    float *X, *Y, *W, *P;
    void fill_scal(float2 *, int) {}          // no optimizer
    static int round(prl_cb *s, prl_buf *buf, int B, cudaStream_t st);
};

static int cb_check(const prl_cb_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim >= 0 && c->action_dim >= 0 && c->obs_dim + c->action_dim >= 1, "obs_dim + action_dim must be positive");
    PRL_REQUIRE(c->obs_dim + c->action_dim + 1 <= kMaxD,
                "obs_dim + action_dim = %d: the ridge solve supports at most %d features (%d with the intercept)",
                c->obs_dim + c->action_dim, kMaxD - 1, kMaxD);
    PRL_REQUIRE(c->action_rep >= 0 && c->action_rep <= 2, "action_rep must be 0 (none), 1 (one-hot) or 2 (binary)");
    PRL_REQUIRE(c->action_rep != 1 || c->action_dim == c->n_actions, "a one-hot representation has action_dim = n_actions");
    PRL_REQUIRE(c->action_rep != 2 || (c->action_dim >= 1 && c->action_dim <= 30 && c->n_actions <= (1 << c->action_dim)),
                "a binary representation needs 1 <= action_dim <= 30 bits and n_actions <= 2^action_dim");
    PRL_REQUIRE(c->l2_reg_lambda > 0.0, "l2_reg_lambda must be positive (A + lambda I must be invertible)");
    PRL_REQUIRE(c->gamma > 0.0 && c->gamma <= 1.0, "gamma must be in (0, 1]");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    PRL_REQUIRE((int64_t)c->max_batch * (c->obs_dim + c->action_dim) < ((int64_t)1 << 31),
                "max_batch * (obs_dim + action_dim) must stay below 2^31 (32-bit element offsets)");
    return PRL_OK;
}

// the workspace, in order; base == null: only its size
static int64_t cb_carve(prl_cb *s, void *base) {
    const prl_cb_cfg &c = s->cfg;
    const int64_t B = c.max_batch, K = c.obs_dim + c.action_dim, chunks = (B + kChunk - 1) / kChunk;
    Carve w{(char *)base};
    w(s->X, B * K); w(s->Y, B); w(s->W, B);
    w(s->P, chunks * cb_entries((int)K + 1));
    s->carve_tail(w, c.max_rounds, B);
    return w.bytes;
}

extern "C" int64_t prl_cb_workspace_bytes(const prl_cb_cfg *c) {
    if (cb_check(c)) return -1;
    prl_cb t; t.cfg = *c;
    return cb_carve(&t, nullptr);
}

extern "C" int prl_cb_create(prl_cb **out, const prl_cb_cfg *cfg, float *A, float *b, float *sum_weight, float *inv_A, float *coefs,
                             double *last_discount, void *workspace) {
    PRL_REQUIRE(out && A && b && sum_weight && inv_A && coefs && last_discount && workspace, "null argument");
    int rc = cb_check(cfg);
    if (rc) return rc;
    const int d = cfg->obs_dim + cfg->action_dim + 1;
    PRL_CUDA(cb_solve_prepare());
    prl_cb *s = new (std::nothrow) prl_cb();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    s->k = d - 1; s->d = d;
    s->A = A; s->b = b; s->sum_weight = sum_weight; s->inv_A = inv_A; s->coefs = coefs; s->last_discount = last_discount;
    cb_carve(s, workspace);
    return prl_cb::open(s, out);
}
extern "C" int prl_cb_destroy(prl_cb *s) { return prl_cb::destroy(s); }
extern "C" int prl_cb_set_graph(prl_cb *s, int enable) { return prl_cb::set_graph(s, enable); }
extern "C" int64_t prl_cb_last_launches(const prl_cb *s) { return prl_cb::last_launches_of(s); }

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
int prl_cb::round(prl_cb *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_cb_cfg &c = s->cfg;
    const int k = s->k, d = s->d, E = cb_entries(d), chunks = (B + kChunk - 1) / kChunk, eb = 256;
    k_cb_load<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf ? buf->records : nullptr, buf ? buf->lay : prl_buf_layout{}, c.obs_dim,
                                                    c.action_dim, c.action_rep, s->call, s->round_idx, B, s->X, s->Y, s->W);
    k_cb_stats<<<dim3(chunks, (E + 255) / 256), 256, 0, st>>>(B, k, s->X, s->Y, s->W, s->P);
    k_cb_reduce<<<(E + eb - 1) / eb, eb, 0, st>>>(d, chunks, s->P, s->A, s->b, s->sum_weight);
    k_cb_solve<<<1, kSolveThreads, cb_solve_smem(d), st>>>(d, (float)c.l2_reg_lambda, (float)c.gamma, c.discount_interval, s->A, s->b,
                                                           s->sum_weight, s->last_discount, s->inv_A, s->coefs, s->round_idx);
    k_cb_predict<<<(B + eb - 1) / eb, eb, 0, st>>>(B, k, s->X, s->Y, s->W, s->coefs, s->call, s->round_idx);
    s->launches_per_round = 5;
    return PRL_OK;
}

extern "C" int prl_cb_learn(prl_cb *s, prl_buf *buf, int rounds, int batch, float *out_pred, float *out_label, float *out_weight,
                            int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && out_pred, "null argument");
    PRL_REQUIRE(s->cfg.action_rep != 0, "learn over a buffer needs a one-hot or binary action representation (action_rep 1 or 2)");
    CbCall call{};
    call.out_pred = out_pred; call.out_label = out_label; call.out_weight = out_weight;
    return prl_cb::learn(s, buf, rounds, batch, 0, out_logical, call, stream_);
}

extern "C" int prl_cb_learn_batch(prl_cb *s, int batch, const float *state, const float *action, const float *reward,
                                  const float *weight, float *out_pred, void *stream_) {
    PRL_REQUIRE(s && (state || s->cfg.obs_dim == 0) && (action || s->cfg.action_dim == 0) && reward && out_pred, "null argument");
    CbCall dense{};
    dense.d_state = state; dense.d_action = action; dense.d_reward = reward; dense.d_weight = weight;
    dense.d_action_ld = s->cfg.action_dim;
    dense.out_pred = out_pred;
    return prl_cb::learn_batch(s, batch, 0, dense, stream_);
}

extern "C" int prl_cb_scores(prl_cb *s, int n, const float *state, int n_space, const float *act_feat, double alpha, int with_sigma,
                             const uint8_t *mask, float *out_scores, int32_t *out_index, void *stream_) {
    PRL_REQUIRE(s && out_scores && (state || s->cfg.obs_dim == 0) && (act_feat || s->cfg.action_dim == 0), "null argument");
    PRL_REQUIRE(n >= 0 && n_space >= 1 && (int64_t)n * n_space < ((int64_t)1 << 31), "n * n_space must be in [0, 2^31)");
    if (n == 0) return PRL_OK;
    const prl_cb_cfg &c = s->cfg;
    cudaStream_t st = (cudaStream_t)stream_;
    const long long rows = (long long)n * n_space;
    k_cb_scores<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(n, n_space, c.obs_dim, c.action_dim, state, act_feat, s->inv_A, s->coefs,
                                                            with_sigma, (float)alpha, out_scores);
    if (out_index) k_cb_argmax<<<(n + 255) / 256, 256, 0, st>>>(n, n_space, out_scores, mask, out_index);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

// no handle: both ridge learners (and a caller holding only the buffers) sample through this one entry
extern "C" int prl_cb_ts_sample(int d, double lam, const float *A, const float *coefs, const float *eps, float *out_theta,
                                int32_t *out_status, void *stream_) {
    PRL_REQUIRE(A && coefs && eps && out_theta && out_status, "null argument");
    PRL_REQUIRE(d >= 1 && d <= kMaxD, "d = %d: the sampler supports 1 <= d <= %d", d, kMaxD);
    PRL_CUDA(cb_solve_prepare());
    PRL_CUDA(cb_ts_sample(d, (float)lam, A, coefs, eps, out_theta, out_status, (cudaStream_t)stream_));
    return PRL_OK;
}

extern "C" int prl_cb_ts_scores(prl_cb *s, int n, const float *state, int n_space, const float *act_feat, const float *theta,
                                const float *z, const uint8_t *mask, float *out_scores, int32_t *out_index, int32_t *out_status,
                                void *stream_) {
    PRL_REQUIRE(s && out_scores && (state || s->cfg.obs_dim == 0) && (act_feat || s->cfg.action_dim == 0), "null argument");
    PRL_REQUIRE((theta != nullptr) != (z != nullptr), "exactly one of theta (sampled coefficients) and z (per-score draws)");
    PRL_REQUIRE(!z || out_status, "the per-score draws need out_status for the NaN-sigma flag");
    PRL_REQUIRE(n >= 0 && n_space >= 1 && (int64_t)n * n_space < ((int64_t)1 << 31), "n * n_space must be in [0, 2^31)");
    cudaStream_t st = (cudaStream_t)stream_;
    if (z) PRL_CUDA(cudaMemsetAsync(out_status, 0, sizeof(int32_t), st));
    if (n == 0) return PRL_OK;
    const prl_cb_cfg &c = s->cfg;
    const long long rows = (long long)n * n_space;
    const unsigned grid = (unsigned)((rows + 7) / 8);
    if (theta)
        k_cb_scores<<<grid, 256, 0, st>>>(n, n_space, c.obs_dim, c.action_dim, state, act_feat, s->inv_A, theta, 0, 0.f, out_scores);
    else
        k_cb_ts_scores<<<grid, 256, 0, st>>>(n, n_space, c.obs_dim, c.action_dim, state, act_feat, s->inv_A, s->coefs, z, out_scores,
                                             out_status);
    if (out_index) k_cb_argmax<<<(n + 255) / 256, 256, 0, st>>>(n, n_space, out_scores, mask, out_index);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}
