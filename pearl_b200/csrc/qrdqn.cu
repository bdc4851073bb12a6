// qrdqn.cu — Quantile Regression DQN (QuantileRegressionDeepQLearning.learn_batch, driven by PolicyLearner.learn or called
// directly on a caller's batch), replacing
//   policy_learners/sequential_decision_making/quantile_regression_deep_td_learning.py   learn_batch (pairwise quantile
//       Huber loss, AdamW step, target update after the step)
//   policy_learners/sequential_decision_making/quantile_regression_deep_q_learning.py    _get_next_state_quantiles
//   neural_networks/sequential_decision_making/q_value_networks.py (QuantileQValueNetwork: mlp_block(state || action) -> N)
//   safety_modules/risk_sensitive_safety_modules.py (RiskNeutralSafetyModule, QuantileNetworkMeanVarianceSafetyModule)
//   utils/functional_utils/learning/loss_fn_utils.py (compute_elementwise_huber_loss, kappa = 1)
//
// One round: the online net at the taken action (one-hot fold, B rows), the target net over every next-action slot (fold
// expanded to B*A rows), the risk-metric greedy slot and the distributional target, the pairwise quantile-Huber gradient,
// the backward pass, AdamW(amsgrad) and, in the rounds whose flag is set, the soft target update with the new parameters.
// Fixed launch sequence, captured once per (batch, buffer) into a CUDA graph and replayed (DESIGN.md §3.4).  The AdamW
// step sizes, the decay factor, the per-round target-update flags and the risk coefficient beta are read through the
// per-call block, so neither prl_qrdqn_set_lr nor a new beta needs a new capture.  fp32, fixed summation order, no float
// atomics: bit-reproducible run to run.
#include <limits.h>
#include <math.h>
#include <stdarg.h>

#include <new>

#include "common.cuh"
#include "rounds.cuh"
#include "gemm.cuh"
#include "qrows.cuh"

using namespace prl;

namespace {

constexpr int kMaxQuantiles = 256;   // k_qr_loss: one thread per quantile of a row
constexpr int kMaxA = 255;           // next-action ids are stored as bytes

// per-call block the captured round reads through
struct QrCall : QSetCall {
    float beta;                               // variance weight of the risk metric (0: risk neutral)
};

// rows of one round (load_row) and the taken action; slots at and beyond the row's count are masked by k_qr_target
__global__ void __launch_bounds__(256, 8) k_qr_load(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int A, int dynamic,
                          const QrCall *__restrict__ call, const int *__restrict__ round_idx, int B, float *__restrict__ S,
                          float *__restrict__ S2, int *__restrict__ act, float *__restrict__ R, float *__restrict__ T,
                          int *__restrict__ cnt, int *__restrict__ ids) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    const QRow row = load_row<true>(records, L, obs, A, dynamic, call, round_idx, B, w, lane, S, S2, R, T, ids);
    if (lane == 0) {
        act[w] = row.action;
        cnt[w] = row.cnt;
    }
}

// Greedy next slot and distributional target (_get_next_state_quantiles, learn_batch step 2).  One warp per row; lane l
// scores slots l, l + 32, ...:
//   rho_k = mean_j q_kj - beta * sum_j w_j (q_kj - mean)^2,  w_j = fl(fl((j + 1) / N) - fl(j / N)),  -inf at k >= count
//   g = first argmax (ties to the lower slot, as torch.argmax);  T_j = q_gj * gamma * (1 - terminated) + r
__global__ void __launch_bounds__(128) k_qr_target(int B, int A, int N, const float *__restrict__ qt, const int *__restrict__ cnt,
                                                   const QrCall *__restrict__ call, float gamma, const float *__restrict__ term,
                                                   const float *__restrict__ rew, float *__restrict__ tq) {
    const int lane = threadIdx.x & 31, b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= B) return;
    const float beta = call->beta, fN = (float)N;
    const int n_ok = cnt[b];
    float best = -INFINITY;
    int bk = INT_MAX;
    for (int k = lane; k < A; k += 32) {
        float rho = -INFINITY;
        if (k < n_ok) {
            const float *q = qt + ((size_t)b * A + k) * N;
            float s = 0.f;
            for (int j = 0; j < N; j++) s = __fadd_rn(s, q[j]);
            const float mean = __fdiv_rn(s, fN);
            float var = 0.f, lo = 0.f;
            for (int j = 0; j < N; j++) {
                const float hi = __fdiv_rn((float)(j + 1), fN), d = __fsub_rn(q[j], mean);
                var = __fadd_rn(var, __fmul_rn(__fsub_rn(hi, lo), __fmul_rn(d, d)));
                lo = hi;
            }
            rho = __fsub_rn(mean, __fmul_rn(beta, var));
        }
        if (rho > best || (rho == best && k < bk)) { best = rho; bk = k; }
    }
    warp_first_max(best, bk);
    const int g = bk == INT_MAX ? 0 : bk;
    const float live = __fsub_rn(1.f, term[b]), r = rew[b];
    const float *q = qt + ((size_t)b * A + g) * N;
    for (int j = lane; j < N; j += 32) tq[(size_t)b * N + j] = __fadd_rn(__fmul_rn(__fmul_rn(q[j], gamma), live), r);
}

// Pairwise quantile-Huber loss (learn_batch steps 3-5) and the reported |theta - T|.  One CTA per row b, thread i < N owns
// theta_i and walks the targets j = 0 .. N-1 in order:
//   u = T_j - theta_i,  w = |tau^_i - 1{u < 0}|,  tau^_i = (i/N + (i+1)/N) / 2,  h'(u) = u if |u| <= 1 else sign(u)
//   L = mean over (b, i) of sum_j w h(u)   ->   dL/dtheta_bi = -sum_j fl(w / (B N)) h'(u)
// rowabs[b] = sum_i |theta_i - T_i| in a fixed tree order.  N <= 256.
__global__ void __launch_bounds__(256) k_qr_loss(int B, int N, const float *__restrict__ theta, const float *__restrict__ tq,
                                                 float *__restrict__ dtheta, float *__restrict__ rowabs) {
    __shared__ float t[kMaxQuantiles], red[256];
    const int b = blockIdx.x, i = threadIdx.x;
    const float fN = (float)N;
    if (i < N) t[i] = tq[(size_t)b * N + i];
    __syncthreads();
    float a = 0.f;
    if (i < N) {
        const float th = theta[(size_t)b * N + i];
        const float tau = __fmul_rn(__fadd_rn(__fdiv_rn((float)(i + 1), fN), __fdiv_rn((float)i, fN)), 0.5f);
        const float g = __fdiv_rn(1.f, (float)(B * N));
        float s = 0.f;
        for (int j = 0; j < N; j++) {
            const float u = __fsub_rn(t[j], th);
            const float w = fabsf(__fsub_rn(tau, u < 0.f ? 1.f : 0.f));
            const float hp = fabsf(u) <= 1.f ? u : copysignf(1.f, u);
            s = __fadd_rn(s, __fmul_rn(__fmul_rn(g, w), hp));
        }
        dtheta[(size_t)b * N + i] = -s;
        a = fabsf(__fsub_rn(th, t[i]));
    }
    red[i] = a;
    __syncthreads();
    for (int o = 128; o; o >>= 1) {
        if (i < o) red[i] += red[i + o];
        __syncthreads();
    }
    if (i == 0) rowabs[b] = red[0];
}

// reported loss mean over B*N of |theta - T| (rows in a fixed tree order), then the round counter advances
__global__ void __launch_bounds__(256) k_qr_report(int B, int N, const float *__restrict__ rowabs, const QrCall *__restrict__ call,
                                                   int *__restrict__ round_idx) {
    __shared__ float red[256];
    float s = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) s += rowabs[b];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        call->out_loss[*round_idx] = red[0] / (float)(B * N);
        *round_idx += 1;
    }
}

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_qrdqn : Rounds<prl_qrdqn, QrCall> {
    static constexpr const char *kFn = "prl_qrdqn", *kName = "QR-DQN";
    static constexpr bool kTargetOn = true;
    static constexpr int kGraphs = 3;
    void fill_call(QrCall &k) const { k.decay = (float)(1.0 - cfg.lr * cfg.weight_decay); }
    prl_qrdqn_cfg cfg;
    int P;
    int W1, b1, W2, b2, W3, b3;
    float *q, *q_m, *q_v, *q_x, *q_t;
    // workspace
    float *S, *S2, *R, *T, *P1, *h1, *h2, *theta, *P1t, *c1t, *c2t, *qt, *tq, *dtheta, *rowabs, *dh2, *dh1, *grad;
    int *act, *cnt, *ids;
    static int round(prl_qrdqn *s, prl_buf *buf, int B, cudaStream_t st);
};

static void qr_layout(prl_qrdqn *s) {
    const prl_qrdqn_cfg &c = s->cfg;
    const int D = c.obs_dim + c.n_actions;
    int o = 0;
    s->W1 = o; o += c.hidden1 * D; s->b1 = o; o += c.hidden1;
    s->W2 = o; o += c.hidden2 * c.hidden1; s->b2 = o; o += c.hidden2;
    s->W3 = o; o += c.num_quantiles * c.hidden2; s->b3 = o; o += c.num_quantiles;
    s->P = o;
}

static int qr_check(const prl_qrdqn_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->hidden1 > 0 && c->hidden2 > 0, "dimensions must be positive");
    PRL_REQUIRE(c->n_actions > 0 && c->n_actions <= kMaxA, "n_actions must be in [1, %d]", kMaxA);
    PRL_REQUIRE(c->num_quantiles > 0 && c->num_quantiles <= kMaxQuantiles, "num_quantiles must be in [1, %d]", kMaxQuantiles);
    PRL_REQUIRE(c->target_update_freq > 0, "target_update_freq must be positive");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    return PRL_OK;
}

extern "C" int64_t prl_qrdqn_param_count(const prl_qrdqn_cfg *c) {
    if (qr_check(c)) return -1;
    prl_qrdqn t; t.cfg = *c; qr_layout(&t);
    return t.P;
}

// the workspace, in order; base == null: only its size
static int64_t qr_carve(prl_qrdqn *s, void *base) {
    const prl_qrdqn_cfg &c = s->cfg;
    const int64_t B = c.max_batch, O = c.obs_dim, A = c.n_actions, N = c.num_quantiles, BA = B * A, H1 = c.hidden1, H2 = c.hidden2;
    Carve w{(char *)base};
    w(s->S, B * O); w(s->S2, B * O); w(s->R, B); w(s->T, B);
    w(s->P1, B * H1); w(s->h1, B * H1); w(s->h2, B * H2); w(s->theta, B * N);          // online, taken action
    w(s->P1t, B * H1); w(s->c1t, BA * H1); w(s->c2t, BA * H2); w(s->qt, BA * N);       // target, every slot
    w(s->tq, B * N); w(s->dtheta, B * N); w(s->rowabs, B);
    w(s->dh2, B * H2); w(s->dh1, B * H1); w(s->grad, s->P);
    w(s->act, B); w(s->cnt, B); w(s->ids, BA);
    s->carve_tail(w, c.max_rounds, B);
    return w.bytes;
}
extern "C" int64_t prl_qrdqn_workspace_bytes(const prl_qrdqn_cfg *c) {
    if (qr_check(c)) return -1;
    prl_qrdqn t; t.cfg = *c; qr_layout(&t);
    return qr_carve(&t, nullptr);
}

extern "C" int prl_qrdqn_create(prl_qrdqn **out, const prl_qrdqn_cfg *cfg, float *q_w, float *q_m, float *q_v, float *q_vmax,
                                float *q_target_w, int64_t adam_step, void *workspace) {
    PRL_REQUIRE(out && q_w && q_m && q_v && q_vmax && q_target_w && workspace, "null argument");
    int rc = qr_check(cfg);
    if (rc) return rc;
    prl_qrdqn *s = new (std::nothrow) prl_qrdqn();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    qr_layout(s);
    s->q = q_w; s->q_m = q_m; s->q_v = q_v; s->q_x = q_vmax; s->q_t = q_target_w;
    s->adam_step = adam_step;
    qr_carve(s, workspace);
    return prl_qrdqn::open(s, out);
}
extern "C" int prl_qrdqn_destroy(prl_qrdqn *s) { return prl_qrdqn::destroy(s); }
extern "C" int64_t prl_qrdqn_adam_step(const prl_qrdqn *s) { return prl_qrdqn::adam_step_of(s); }
extern "C" int prl_qrdqn_set_lr(prl_qrdqn *s, double lr) { return prl_qrdqn::set_lr(s, lr); }
extern "C" int prl_qrdqn_set_graph(prl_qrdqn *s, int enable) { return prl_qrdqn::set_graph(s, enable); }
extern "C" int64_t prl_qrdqn_last_launches(const prl_qrdqn *s) { return prl_qrdqn::last_launches_of(s); }

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
int prl_qrdqn::round(prl_qrdqn *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_qrdqn_cfg &c = s->cfg;
    const int O = c.obs_dim, A = c.n_actions, D = O + A, N = c.num_quantiles, H1 = c.hidden1, H2 = c.hidden2, BA = B * A;
    // the decay factor is overridden by call->decay (k_adamw's decay pointer)
    const AdamHp h = adam_hp(0.0, c.beta1, c.beta2, c.eps, c.weight_decay);
    GemmLauncher L; L.st = st;
    const float *w = s->q, *t = s->q_t;
    float *g = s->grad;
    const int eb = 256;
    int small = 0;
    const int dynamic = (buf && (buf->desc.flags & PRL_BUF_DYNAMIC_ACTIONS)) ? 1 : 0;
    k_qr_load<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf ? buf->records : nullptr, buf ? buf->lay : prl_buf_layout{}, O, A, dynamic,
                                                    s->call, s->round_idx, B, s->S, s->S2, s->act, s->R, s->T, s->cnt, s->ids);
    small++;
    // ---------------- online net at the taken action (kept for the backward pass)
    L.fwd(mat(s->S, O), B, w + s->W1, D, 0, w + s->b1, 0, H1, O, false, s->P1, H1, 0);
    k_fold<<<(B * H1 + eb - 1) / eb, eb, 0, st>>>(B, H1, s->P1, w + s->W1 + O, D, 0, s->act, s->h1);
    L.fwd(mat(s->h1, H1), B, w + s->W2, H1, 0, w + s->b2, 0, H2, H1, true, s->h2, H2, 0);
    L.fwd(mat(s->h2, H2), B, w + s->W3, H2, 0, w + s->b3, 0, N, H2, false, s->theta, N, 0);
    small++;
    // ---------------- target net over every next-action slot: B*A rows of N quantiles
    L.fwd(mat(s->S2, O), B, t + s->W1, D, 0, t + s->b1, 0, H1, O, false, s->P1t, H1, 0);
    k_fold_expand<<<(unsigned)(((long long)BA * H1 + eb - 1) / eb), eb, 0, st>>>(B, A, H1, s->P1t, t + s->W1 + O, D, 0, s->ids, s->c1t);
    L.fwd(mat(s->c1t, H1), BA, t + s->W2, H1, 0, t + s->b2, 0, H2, H1, true, s->c2t, H2, 0);
    L.fwd(mat(s->c2t, H2), BA, t + s->W3, H2, 0, t + s->b3, 0, N, H2, false, s->qt, N, 0);
    small++;
    // ---------------- greedy slot under the risk metric, target quantiles, pairwise quantile-Huber gradient
    k_qr_target<<<(B * 32 + 127) / 128, 128, 0, st>>>(B, A, N, s->qt, s->cnt, s->call, (float)c.gamma, s->T, s->R, s->tq);
    k_qr_loss<<<B, 256, 0, st>>>(B, N, s->theta, s->tq, s->dtheta, s->rowabs);
    small += 2;
    // ---------------- backward through the online net
    L.bwd_w(s->dtheta, N, 0, B, N, mat(s->h2, H2), H2, g + s->W3, H2, 0, g + s->b3, 0);
    L.bwd_x(s->dtheta, N, 0, B, N, w + s->W3, H2, 0, 0, H2, s->dh2, H2, 0, s->h2, H2, 0, false);
    L.bwd_w(s->dh2, H2, 0, B, H2, mat(s->h1, H1), H1, g + s->W2, H1, 0, g + s->b2, 0);
    L.bwd_x(s->dh2, H2, 0, B, H2, w + s->W2, H1, 0, 0, H1, s->dh1, H1, 0, s->h1, H1, 0, false);
    L.bwd_w(s->dh1, H1, 0, B, H1, mat(s->S, O), O, g + s->W1, D, 0, g + s->b1, 0);                   // state columns + b1
    k_fold_w1a_grad<<<(H1 * A + eb - 1) / eb, eb, 0, st>>>(B, A, H1, s->act, s->dh1, g + s->W1 + O, D, 0);
    small++;
    // ---------------- AdamW(amsgrad), then the soft target update with the NEW parameters in flagged rounds
    k_adamw<<<(s->P + eb - 1) / eb, eb, 0, st>>>(s->P, s->q, s->q_m, s->q_v, s->q_x, g, h, s->scal, s->round_idx, s->q_t, (float)c.tau,
                                                (float)(1.0 - c.tau), &s->call->decay, s->target_on);
    k_qr_report<<<1, 256, 0, st>>>(B, N, s->rowabs, s->call, s->round_idx);
    small += 2;
    s->launches_per_round = L.count + small;
    return PRL_OK;
}

extern "C" int prl_qrdqn_learn(prl_qrdqn *s, prl_buf *buf, int rounds, int batch, int64_t training_steps, double beta, float *out_loss,
                               int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && out_loss, "null argument");
    QrCall call{};
    call.beta = (float)beta; call.out_loss = out_loss;
    return prl_qrdqn::learn(s, buf, rounds, batch, training_steps, out_logical, call, stream_);
}

extern "C" int prl_qrdqn_learn_batch(prl_qrdqn *s, int batch, const float *state, const int32_t *action_id, const float *reward,
                                     const float *next_state, const uint8_t *terminated, const int32_t *next_ids,
                                     const int32_t *next_count, int64_t training_steps, double beta, float *out_loss, void *stream_) {
    PRL_REQUIRE(s && state && action_id && reward && next_state && terminated && out_loss, "null argument");
    QrCall dense{};
    dense.d_state = state; dense.d_next_state = next_state; dense.d_reward = reward; dense.d_action_id = action_id;
    dense.d_next_ids = next_ids; dense.d_next_cnt = next_count; dense.d_term = terminated;
    dense.beta = (float)beta;
    dense.out_loss = out_loss;
    return prl_qrdqn::learn_batch(s, batch, training_steps, dense, stream_);
}
