// disjoint_bandit.cu — Pearl's disjoint linear bandits, one ridge regression per arm, all arms in each launch, replacing
//   policy_learners/contextual_bandits/disjoint_bandit.py         DisjointBanditContainer of LinearBandit arms:
//       _validate_batch / _partition_batch_by_arm (a row belongs to arm `action`; an arm without rows gets the null batch,
//       one zero row of weight 0, and still runs its learn_batch), learn_batch (each arm's LinearBandit.learn_batch,
//       _maybe_apply_discounting on the arm's own sum_weight, prediction = model(x) after the update), act / get_scores
//   policy_learners/contextual_bandits/disjoint_linear_bandit.py  DisjointLinearBandit: learn_batch (rows with action ==
//       k to arm k, x = state or state || space[k]; rows of no arm dropped; an arm without rows skipped, no solve), act
//   exploration_modules/contextual_bandits/ucb_exploration.py     DisjointUCBExploration (mu_k + alpha sigma_k, NaN -> 0)
//   exploration_modules/contextual_bandits/thompson_sampling_exploration.py   ThompsonSamplingExplorationLinearDisjoint
//       (one MultivariateNormal(coefs_k, precision = A_k + lambda_k I) draw per arm; the scores stacked (K, n) arm-major)
// on top of LinearRegression (neural_networks/contextual_bandit/linear_regression.py), as bandit.cu.
//
// Round (7 launches, 6 for DisjointLinearBandit, which reports nothing; captured once per (batch, buffer) into a CUDA
// graph and replayed, DESIGN.md §3.6b):
//   k_dj_hist     each row's arm (the stored id, or the caller's id; an id outside [0, K) marks the row dropped) and each
//                 chunk of kChunk rows' per-arm row counts (integer shared-memory counts)
//   k_dj_scan     one CTA, a thread per arm: the arm's rows over the chunks in ascending order, then block scans over the
//                 arms: row offsets, statistic-chunk offsets and report offsets; the chunk table (arm of each chunk)
//   k_dj_rows     the stable partition: each chunk's rows ranked in ascending order by one warp (match_any), then loaded
//                 at their partitioned position as x = state (the arm's slice of a 3-D state) [|| action features of the arm]
//   k_dj_stats    ridge.cuh's statistics body over each arm's chunks of kChunk rows, one chunk per CTA column
//   k_dj_reduce   ridge.cuh's reduction body, one CTA row per arm: each arm's chunks in ascending order into A_k, b_k, sw_k
//   k_dj_solve    one CTA per arm, all arms in one launch: the skip rule, then ridge.cuh's discounting decision and fp64
//                 Gauss-Jordan solve with the arm's lambda, gamma, interval and last_discount
//   k_dj_predict  (container) prediction = [1, x] . coefs_k after the update, label and weight, in partition order with
//                 one row (coefs_k[0], 0, 0) for each arm that had no rows
// No float atomics and a fixed summation order: bit-reproducible run to run, graph or eager, and however the rounds are
// split into calls.  The numerics of each arm are bandit.cu's.
#include <math.h>

#include <new>

#include "common.cuh"
#include "ridge.cuh"
#include "rounds.cuh"

using namespace prl;

namespace {

constexpr int kMaxArms = 1024;      // k_dj_scan's one CTA has a thread per arm

// per-call block the captured round reads through
struct DcbCall {
    const int32_t *slots;                       // [rounds][B] (learn)
    float *out_pred, *out_label, *out_weight;   // [rounds][B + K] report rows (container; may be null)
    int32_t *out_counts;                        // [rounds][K] rows per arm (may be null)
    // learn_batch: the caller's dense batch
    const float *d_state, *d_reward, *d_weight; // d_weight may be null: every weight is 1
    const int32_t *d_arm;
    int d_state3d;                              // d_state is [B][K][obs]: arm k reads its slice
};

__global__ void __launch_bounds__(256) k_dj_hist(const uint32_t *__restrict__ records, prl_buf_layout L, const DcbCall *__restrict__ call,
                                                 const int *__restrict__ round_idx, int B, int K, int *__restrict__ arm,
                                                 int *__restrict__ H) {
    __shared__ int h[kMaxArms];
    for (int a = threadIdx.x; a < K; a += blockDim.x) h[a] = 0;
    __syncthreads();
    const int r = blockIdx.x * kChunk + threadIdx.x;
    if (r < B) {
        int id;
        if (records) {
            const int32_t *slots = call->slots + (size_t)(*round_idx) * B;
            id = (int)records[(size_t)slots[r] * L.record_words + L.off_action];
        } else {
            id = call->d_arm[r];
        }
        const int a = id >= 0 && id < K ? id : K;
        arm[r] = a;
        if (a < K) atomicAdd(&h[a], 1);
    }
    __syncthreads();
    for (int a = threadIdx.x; a < K; a += blockDim.x) H[(size_t)blockIdx.x * K + a] = h[a];
}

// exclusive prefix of v over the CTA's threads (blockDim.x <= 1024), and the total; sh holds blockDim.x ints
__device__ int dj_scan(int v, int *sh, int &total) {
    const int t = threadIdx.x;
    __syncthreads();
    sh[t] = v;
    __syncthreads();
    for (int o = 1; o < (int)blockDim.x; o <<= 1) {
        const int u = t >= o ? sh[t - o] : 0;
        __syncthreads();
        sh[t] += u;
        __syncthreads();
    }
    total = sh[blockDim.x - 1];
    return sh[t] - v;
}

// H[c][k] becomes the rows of arm k in chunks before c; off[k] (off[K] = rows kept), cfirst[k] = the arm's first statistic
// chunk, roff[k] = its first report row (an arm without rows reports one), tab[chunk] = its arm, *ntab = chunks
__global__ void __launch_bounds__(kMaxArms) k_dj_scan(int C, int K, int *__restrict__ H, int *__restrict__ counts, int *__restrict__ off,
                                                      int *__restrict__ cfirst, int *__restrict__ roff, int *__restrict__ tab,
                                                      int *__restrict__ ntab, const DcbCall *__restrict__ call,
                                                      const int *__restrict__ round_idx) {
    __shared__ int sh[kMaxArms];
    const int k = threadIdx.x;
    int n = 0;
    if (k < K)
        for (int c = 0; c < C; c++) {
            const int t = H[(size_t)c * K + k];
            H[(size_t)c * K + k] = n;
            n += t;
        }
    const int nch = (n + kChunk - 1) / kChunk;
    int rows, chunks, reps;
    const int o = dj_scan(n, sh, rows);
    const int cf = dj_scan(nch, sh, chunks);
    const int ro = dj_scan(k < K ? max(n, 1) : 0, sh, reps);
    if (k < K) {
        counts[k] = n; off[k] = o; cfirst[k] = cf; roff[k] = ro;
        if (call->out_counts) call->out_counts[(size_t)(*round_idx) * K + k] = n;
        for (int j = 0; j < nch; j++) tab[cf + j] = k;
    }
    if (k == 0) { off[K] = rows; *ntab = chunks; }
}

// the stable partition and the row load: chunk blockIdx.x's rows ranked within their arm in ascending order by warp 0,
// then each row loaded by one warp at its position off[a] + (rows of a in earlier chunks) + rank
__global__ void __launch_bounds__(256) k_dj_rows(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int adim,
                                                 const float *__restrict__ act_feat, const DcbCall *__restrict__ call,
                                                 const int *__restrict__ round_idx, int B, int K, const int *__restrict__ arm,
                                                 const int *__restrict__ H, const int *__restrict__ off, float *__restrict__ X,
                                                 float *__restrict__ Y, float *__restrict__ W, int *__restrict__ parm) {
    __shared__ int cnt[kMaxArms], pos[kChunk];
    const int lane = threadIdx.x & 31, wb = threadIdx.x >> 5, r0 = blockIdx.x * kChunk;
    for (int a = threadIdx.x; a < K; a += blockDim.x) cnt[a] = 0;
    __syncthreads();
    if (wb == 0)
        for (int g = 0; g < kChunk; g += 32) {
            const int r = r0 + g + lane;
            const int a = r < B ? arm[r] : K;
            const unsigned m = __match_any_sync(0xffffffffu, a);
            const int rank = __popc(m & ((1u << lane) - 1u));
            pos[g + lane] = a < K ? off[a] + H[(size_t)blockIdx.x * K + a] + cnt[a] + rank : -1;
            __syncwarp();
            if (a < K && rank == 0) cnt[a] += __popc(m);
            __syncwarp();
        }
    __syncthreads();
    const int kk = obs + adim;
    const int32_t *slots = records ? call->slots + (size_t)(*round_idx) * B : nullptr;
    for (int lr = wb; lr < kChunk && r0 + lr < B; lr += blockDim.x >> 5) {
        const int p = pos[lr], r = r0 + lr;
        if (p < 0) continue;
        const int a = arm[r];
        float *x = X + (size_t)p * kk;
        if (records) {
            const uint32_t *rec = records + (size_t)slots[r] * L.record_words;
            for (int c = lane; c < obs; c += 32) x[c] = __uint_as_float(rec[L.off_state + c]);
            if (lane == 0) { Y[p] = __uint_as_float(rec[L.off_reward]); W[p] = 1.f; }
        } else {
            const float *st = call->d_state + (call->d_state3d ? ((size_t)r * K + a) * obs : (size_t)r * obs);
            for (int c = lane; c < obs; c += 32) x[c] = st[c];
            if (lane == 0) { Y[p] = call->d_reward[r]; W[p] = call->d_weight ? call->d_weight[r] : 1.f; }
        }
        for (int c = lane; c < adim; c += 32) x[obs + c] = act_feat[(size_t)a * adim + c];
        if (lane == 0) parm[p] = a;
    }
}

// chunk blockIdx.x of the table: rows [j kChunk, +kChunk) of its arm's segment, j = blockIdx.x - cfirst[arm]
__global__ void __launch_bounds__(256) k_dj_stats(int kk, const int *__restrict__ ntab, const int *__restrict__ tab,
                                                  const int *__restrict__ counts, const int *__restrict__ off,
                                                  const int *__restrict__ cfirst, const float *__restrict__ X,
                                                  const float *__restrict__ Y, const float *__restrict__ W, float *__restrict__ P) {
    if ((int)blockIdx.x >= *ntab) return;
    const int a = tab[blockIdx.x], o = off[a], E = cb_entries(kk + 1);
    cb_stats_chunk(counts[a], kk, X + (size_t)o * kk, Y + o, W + o, P + (size_t)cfirst[a] * E, cfirst[a]);
}

// arm blockIdx.y's chunks into A_k, b_k, sum_weight_k (an arm of the container without rows adds zeros, as its null batch
// does; DisjointLinearBandit skips it)
__global__ void __launch_bounds__(256) k_dj_reduce(int d, int skip_empty, const int *__restrict__ counts, const int *__restrict__ cfirst,
                                                   const float *__restrict__ P, float *__restrict__ A, float *__restrict__ b,
                                                   float *__restrict__ sum_weight) {
    const int a = blockIdx.y, n = counts[a];
    if (skip_empty && n == 0) return;
    cb_reduce_entry(d, (n + kChunk - 1) / kChunk, P + (size_t)cfirst[a] * cb_entries(d), A + (size_t)a * d * d, b + (size_t)a * d,
                    sum_weight + a);
}

// one CTA per arm: the arm's discounting decision and solve.  round_idx advances first (no CTA here reads it)
__global__ void __launch_bounds__(kSolveThreads) k_dj_solve(int d, int skip_empty, const int *__restrict__ counts, const float *__restrict__ lam,
                                                            const float *__restrict__ gamma, const double *__restrict__ interval,
                                                            float *__restrict__ A, float *__restrict__ b, const float *__restrict__ sum_weight,
                                                            double *__restrict__ last, float *__restrict__ inv_A, float *__restrict__ coefs,
                                                            int *__restrict__ round_idx) {
    const int a = blockIdx.x;
    if (a == 0 && threadIdx.x == 0) *round_idx += 1;
    if (skip_empty && counts[a] == 0) return;
    const size_t dd = (size_t)d * d;
    cb_solve_ridge(d, lam[a], gamma[a], interval[a], A + a * dd, b + (size_t)a * d, sum_weight + a, last + a, inv_A + a * dd,
                   coefs + (size_t)a * d);
}

// the container's report of the round k_dj_solve finished, row q = roff[arm] + rank in the arm: [1, x] . coefs_arm, label,
// weight; thread B + k writes arm k's null-batch row (prediction [1, 0] . coefs_k = coefs_k[0], label 0, weight 0)
__global__ void __launch_bounds__(256) k_dj_predict(int B, int K, int kk, const int *__restrict__ counts, const int *__restrict__ off,
                                                    const int *__restrict__ roff, const int *__restrict__ parm, const float *__restrict__ X,
                                                    const float *__restrict__ Y, const float *__restrict__ W,
                                                    const float *__restrict__ coefs, const DcbCall *__restrict__ call,
                                                    const int *__restrict__ round_idx) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x, d = kk + 1;
    if (!call->out_pred || t >= B + K) return;
    const size_t base = (size_t)(*round_idx - 1) * (B + K);
    float s, y, w;
    size_t q;
    if (t < B) {
        if (t >= off[K]) return;
        const int a = parm[t];
        const float *x = X + (size_t)t * kk, *c = coefs + (size_t)a * d;
        s = c[0];
        for (int j = 0; j < kk; j++) s = fmaf(x[j], c[j + 1], s);
        y = Y[t]; w = W[t];
        q = base + roff[a] + (t - off[a]);
    } else {
        const int a = t - B;
        if (counts[a] > 0) return;
        s = coefs[(size_t)a * d]; y = 0.f; w = 0.f;
        q = base + roff[a];
    }
    call->out_pred[q] = s;
    if (call->out_label) call->out_label[q] = y;
    if (call->out_weight) call->out_weight[q] = w;
}

// scores of n states x K arms, one warp per (state, arm) row x = [1, state, action features of the arm] on the arm's
// ridge (ridge.cuh's cb_row_form): with_sigma mu + alpha sigma (NaN sigma -> 0), else mu.  Written at s K + k, or with
// arm_major at k n + s: ThompsonSamplingExplorationLinearDisjoint stacks the per-arm scores (K, n) and views them (n, K).
__global__ void __launch_bounds__(256) k_dj_scores(int n, int K, int obs, int adim, const float *__restrict__ state,
                                                   const float *__restrict__ act_feat, const float *__restrict__ inv_A,
                                                   const float *__restrict__ coefs, int with_sigma, float alpha, int arm_major,
                                                   float *__restrict__ out) {
    __shared__ float xs[8][kMaxD];
    const int lane = threadIdx.x & 31, wb = threadIdx.x >> 5, d = obs + adim + 1;
    const long long row = (long long)blockIdx.x * 8 + wb;
    if (row >= (long long)n * K) return;
    const int s = (int)(row / K), a = (int)(row - (long long)s * K);
    float mu, q;
    cb_row_form(s, a, obs, adim, state, act_feat, inv_A + (size_t)a * d * d, coefs + (size_t)a * d, with_sigma, xs[wb], lane, mu, q);
    if (lane == 0) {
        float v = mu;
        if (with_sigma) {
            float sg = sqrtf(q);
            if (isnan(sg)) sg = 0.f;
            v = __fadd_rn(mu, __fmul_rn(alpha, sg));
        }
        out[arm_major ? (size_t)a * n + s : (size_t)row] = v;
    }
}

// one CTA per arm: ridge.cuh's sampler on the arm's A_k + lambda_k I, coefs_k and draws eps[k][d]; status[k] = 0, or 1
// when the arm's precision matrix is not positive definite
__global__ void __launch_bounds__(kSolveThreads) k_dj_ts_sample(int d, const float *__restrict__ lam, const float *__restrict__ A,
                                                                const float *__restrict__ coefs, const float *__restrict__ eps,
                                                                float *__restrict__ theta, int *__restrict__ status) {
    const int a = blockIdx.x;
    const size_t o = (size_t)a * d;
    cb_ts_draw(d, lam[a], A + o * d, coefs + o, eps + o, theta + o, status + a);
}

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_dcb : Rounds<prl_dcb, DcbCall> {
    static constexpr const char *kFn = "prl_dcb", *kName = "DisjointBandit";
    prl_dcb_cfg cfg;
    int K, kk, d;
    float *A, *b, *sum_weight, *inv_A, *coefs;
    const float *lam, *gamma, *act_feat;
    const double *interval;
    double *last;
    int *arm, *parm, *H, *counts, *off, *cfirst, *roff, *tab, *ntab;
    float *X, *Y, *W, *P;
    void fill_scal(float2 *, int) {}          // no optimizer
    static int round(prl_dcb *s, prl_buf *buf, int B, cudaStream_t st);
    // stored ids index the arms: a buffer of up to K actions
    int buffer_ok(const prl_buf *buf) const {
        PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.obs_dim == cfg.obs_dim && buf->desc.n_actions <= K,
                    "%s needs a discrete-action buffer with obs_dim = %d and n_actions <= %d arms", kName, cfg.obs_dim, K);
        PRL_REQUIRE(buf->shard_world <= 1, "the buffer is one shard of a multi-GPU buffer: %s samples local buffers only", kName);
        return PRL_OK;
    }
};

static int dcb_check(const prl_dcb_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->mode == 0 || c->mode == 1, "mode must be 0 (DisjointBanditContainer) or 1 (DisjointLinearBandit)");
    PRL_REQUIRE(c->n_arms >= 1 && c->n_arms <= kMaxArms, "n_arms = %d: the disjoint learner supports 1 to %d arms", c->n_arms, kMaxArms);
    PRL_REQUIRE(c->obs_dim >= 0 && c->action_dim >= 0 && c->obs_dim + c->action_dim >= 1, "obs_dim + action_dim must be positive");
    PRL_REQUIRE(c->mode == 1 || c->action_dim == 0, "the container's arms read the state alone (action_dim 0)");
    PRL_REQUIRE(c->obs_dim + c->action_dim + 1 <= kMaxD,
                "obs_dim + action_dim = %d: the ridge solve supports at most %d features (%d with the intercept)",
                c->obs_dim + c->action_dim, kMaxD - 1, kMaxD);
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    PRL_REQUIRE((int64_t)c->max_batch * (c->obs_dim + c->action_dim) < ((int64_t)1 << 31),
                "max_batch * (obs_dim + action_dim) must stay below 2^31 (32-bit element offsets)");
    return PRL_OK;
}

// the workspace, in order; base == null: only its size
static int64_t dcb_carve(prl_dcb *s, void *base) {
    const prl_dcb_cfg &c = s->cfg;
    const int64_t B = c.max_batch, K = c.n_arms, kk = c.obs_dim + c.action_dim, C = (B + kChunk - 1) / kChunk;
    const int64_t maxch = C + (K < B ? K : B);
    Carve w{(char *)base};
    w(s->arm, B); w(s->parm, B); w(s->H, C * K); w(s->counts, K); w(s->off, K + 1); w(s->cfirst, K); w(s->roff, K);
    w(s->tab, maxch); w(s->ntab, 1);
    w(s->X, B * kk); w(s->Y, B); w(s->W, B);
    w(s->P, maxch * cb_entries((int)kk + 1));
    s->carve_tail(w, c.max_rounds, B);
    return w.bytes;
}

static cudaError_t dcb_prepare() {
    const int smem = (int)cb_solve_smem(kMaxD);
    const cudaError_t e = cudaFuncSetAttribute(k_dj_solve, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(k_dj_ts_sample, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
}

// disjoint_bandit.py / disjoint_linear_bandit.py __init__: the arms' LinearRegression buffers as flat arrays
extern "C" int64_t prl_dcb_workspace_bytes(const prl_dcb_cfg *c) {
    if (dcb_check(c)) return -1;
    prl_dcb t; t.cfg = *c;
    return dcb_carve(&t, nullptr);
}

extern "C" int prl_dcb_create(prl_dcb **out, const prl_dcb_cfg *cfg, float *A, float *b, float *sum_weight, float *inv_A, float *coefs,
                              const float *lam, const float *gamma, const double *interval, double *last, const float *act_feat,
                              void *workspace) {
    PRL_REQUIRE(out && A && b && sum_weight && inv_A && coefs && lam && gamma && interval && last && workspace, "null argument");
    int rc = dcb_check(cfg);
    if (rc) return rc;
    PRL_REQUIRE(act_feat || cfg->action_dim == 0, "null act_feat with action_dim > 0");
    PRL_CUDA(dcb_prepare());
    prl_dcb *s = new (std::nothrow) prl_dcb();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    s->K = cfg->n_arms; s->kk = cfg->obs_dim + cfg->action_dim; s->d = s->kk + 1;
    s->A = A; s->b = b; s->sum_weight = sum_weight; s->inv_A = inv_A; s->coefs = coefs;
    s->lam = lam; s->gamma = gamma; s->interval = interval; s->last = last; s->act_feat = act_feat;
    dcb_carve(s, workspace);
    return prl_dcb::open(s, out);
}
extern "C" int prl_dcb_destroy(prl_dcb *s) { return prl_dcb::destroy(s); }
extern "C" int prl_dcb_set_graph(prl_dcb *s, int enable) { return prl_dcb::set_graph(s, enable); }
extern "C" int64_t prl_dcb_last_launches(const prl_dcb *s) { return prl_dcb::last_launches_of(s); }

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
int prl_dcb::round(prl_dcb *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_dcb_cfg &c = s->cfg;
    const int K = s->K, kk = s->kk, d = s->d, E = cb_entries(d), C = (B + kChunk - 1) / kChunk, maxch = C + (K < B ? K : B);
    const int skip = c.mode == 1;
    const uint32_t *rec = buf ? buf->records : nullptr;
    const prl_buf_layout L = buf ? buf->lay : prl_buf_layout{};
    k_dj_hist<<<C, kChunk, 0, st>>>(rec, L, s->call, s->round_idx, B, K, s->arm, s->H);
    k_dj_scan<<<1, kMaxArms, 0, st>>>(C, K, s->H, s->counts, s->off, s->cfirst, s->roff, s->tab, s->ntab, s->call, s->round_idx);
    k_dj_rows<<<C, 256, 0, st>>>(rec, L, c.obs_dim, c.action_dim, s->act_feat, s->call, s->round_idx, B, K, s->arm, s->H, s->off,
                                 s->X, s->Y, s->W, s->parm);
    k_dj_stats<<<dim3(maxch, (E + 255) / 256), 256, 0, st>>>(kk, s->ntab, s->tab, s->counts, s->off, s->cfirst, s->X, s->Y, s->W, s->P);
    k_dj_reduce<<<dim3((E + 255) / 256, K), 256, 0, st>>>(d, skip, s->counts, s->cfirst, s->P, s->A, s->b, s->sum_weight);
    k_dj_solve<<<K, kSolveThreads, cb_solve_smem(d), st>>>(d, skip, s->counts, s->lam, s->gamma, s->interval, s->A, s->b, s->sum_weight,
                                                          s->last, s->inv_A, s->coefs, s->round_idx);
    s->launches_per_round = 6;
    if (c.mode == 0) {
        k_dj_predict<<<(B + K + 255) / 256, 256, 0, st>>>(B, K, kk, s->counts, s->off, s->roff, s->parm, s->X, s->Y, s->W, s->coefs,
                                                          s->call, s->round_idx);
        s->launches_per_round = 7;
    }
    return PRL_OK;
}

// PolicyLearner.learn (policy_learner.py:162-195) over the container's / DisjointLinearBandit's learn_batch
extern "C" int prl_dcb_learn(prl_dcb *s, prl_buf *buf, int rounds, int batch, float *out_pred, float *out_label, float *out_weight,
                             int32_t *out_counts, int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf, "null argument");
    DcbCall call{};
    call.out_pred = out_pred; call.out_label = out_label; call.out_weight = out_weight; call.out_counts = out_counts;
    return prl_dcb::learn(s, buf, rounds, batch, 0, out_logical, call, stream_);
}

// DisjointBanditContainer.learn_batch (disjoint_bandit.py:67-161) / DisjointLinearBandit.learn_batch
// (disjoint_linear_bandit.py:69-116) on a dense device batch
extern "C" int prl_dcb_learn_batch(prl_dcb *s, int batch, const float *state, int state3d, const int32_t *arm, const float *reward,
                                   const float *weight, float *out_pred, float *out_label, float *out_weight, int32_t *out_counts,
                                   void *stream_) {
    PRL_REQUIRE(s && (state || s->cfg.obs_dim == 0) && arm && reward, "null argument");
    DcbCall dense{};
    dense.d_state = state; dense.d_state3d = state3d != 0; dense.d_arm = arm; dense.d_reward = reward; dense.d_weight = weight;
    dense.out_pred = out_pred; dense.out_label = out_label; dense.out_weight = out_weight; dense.out_counts = out_counts;
    return prl_dcb::learn_batch(s, batch, 0, dense, stream_);
}

// DisjointBanditContainer.get_scores / act with DisjointUCBExploration (ucb_exploration.py:122-155; disjoint_bandit.py:171-239,
// ensemble_forward), and exploit's mu alone (with_sigma 0)
extern "C" int prl_dcb_scores(prl_dcb *s, int n, const float *state, const float *act_feat, double alpha, int with_sigma,
                              const uint8_t *mask, float *out_scores, int32_t *out_index, void *stream_) {
    PRL_REQUIRE(s && out_scores && (state || s->cfg.obs_dim == 0) && (act_feat || s->cfg.action_dim == 0), "null argument");
    PRL_REQUIRE(n >= 0 && (int64_t)n * s->K < ((int64_t)1 << 31), "n * n_arms must be in [0, 2^31)");
    if (n == 0) return PRL_OK;
    cudaStream_t st = (cudaStream_t)stream_;
    const long long rows = (long long)n * s->K;
    k_dj_scores<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(n, s->K, s->cfg.obs_dim, s->cfg.action_dim, state, act_feat, s->inv_A,
                                                            s->coefs, with_sigma, (float)alpha, 0, out_scores);
    if (out_index) k_cb_argmax<<<(n + 255) / 256, 256, 0, st>>>(n, s->K, out_scores, mask, out_index);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

// ThompsonSamplingExplorationLinearDisjoint.get_scores (thompson_sampling_exploration.py:117-142): one MultivariateNormal
// draw per arm (lines 63-68), all arms in one launch
extern "C" int prl_dcb_ts_sample(prl_dcb *s, const float *eps, float *out_theta, int32_t *out_status, void *stream_) {
    PRL_REQUIRE(s && eps && out_theta && out_status, "null argument");
    k_dj_ts_sample<<<s->K, kSolveThreads, cb_solve_smem(s->d), (cudaStream_t)stream_>>>(s->d, s->lam, s->A, s->coefs, eps, out_theta,
                                                                                       out_status);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

// the Thompson scores x1 . theta_k (lines 69-74) in the reference's arm-major layout (line 141-142), and the first maximum
extern "C" int prl_dcb_ts_scores(prl_dcb *s, int n, const float *state, const float *act_feat, const float *theta, const uint8_t *mask,
                                 float *out_scores, int32_t *out_index, void *stream_) {
    PRL_REQUIRE(s && theta && out_scores && (state || s->cfg.obs_dim == 0) && (act_feat || s->cfg.action_dim == 0), "null argument");
    PRL_REQUIRE(n >= 0 && (int64_t)n * s->K < ((int64_t)1 << 31), "n * n_arms must be in [0, 2^31)");
    if (n == 0) return PRL_OK;
    cudaStream_t st = (cudaStream_t)stream_;
    const long long rows = (long long)n * s->K;
    k_dj_scores<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(n, s->K, s->cfg.obs_dim, s->cfg.action_dim, state, act_feat, s->inv_A,
                                                            theta, 0, 0.f, 1, out_scores);
    if (out_index) k_cb_argmax<<<(n + 255) / 256, 256, 0, st>>>(n, s->K, out_scores, mask, out_index);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}
