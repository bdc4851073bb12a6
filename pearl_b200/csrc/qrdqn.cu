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
#include "gemm.cuh"

using namespace prl;

namespace {

constexpr int kMaxQuantiles = 256;   // k_qr_loss: one thread per quantile of a row
constexpr int kMaxA = 255;           // next-action ids are stored as bytes

// per-call block the captured round reads through
struct QrCall {
    const int32_t *slots;                     // [rounds][B] (learn)
    float *out_loss;                          // [rounds]
    // learn_batch: the caller's dense batch
    const float *d_state, *d_next_state, *d_reward;
    const int32_t *d_action_id, *d_next_ids, *d_next_cnt;   // next ids / counts may be null: every action available
    const uint8_t *d_term;
    float decay;                              // AdamW decoupled decay 1 - lr * weight_decay
    float beta;                               // variance weight of the risk metric (0: risk neutral)
};

// rows of one round: state, next state, action id, reward, terminated, and the next-action id of every slot (slot k holds
// id_k; slots at and beyond the row's count are masked by k_qr_target).  records == null: pack the caller's dense batch.
__global__ void k_qr_load(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int A, int dynamic,
                          const QrCall *__restrict__ call, const int *__restrict__ round_idx, int B, float *__restrict__ S,
                          float *__restrict__ S2, int *__restrict__ act, float *__restrict__ R, float *__restrict__ T,
                          int *__restrict__ cnt, int *__restrict__ ids) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    if (!records) {
        for (int p = lane; p < obs; p += 32) {
            S[(size_t)w * obs + p] = call->d_state[(size_t)w * obs + p];
            S2[(size_t)w * obs + p] = call->d_next_state[(size_t)w * obs + p];
        }
        const int32_t *nid = call->d_next_ids;
        for (int k = lane; k < A; k += 32) ids[(size_t)w * A + k] = nid ? nid[(size_t)w * A + k] : k;
        if (lane == 0) {
            act[w] = call->d_action_id[w];
            R[w] = call->d_reward[w];
            T[w] = call->d_term[w] ? 1.f : 0.f;
            cnt[w] = call->d_next_cnt ? min(call->d_next_cnt[w], A) : A;
        }
        return;
    }
    const int32_t *slots = call->slots + (size_t)(*round_idx) * B;
    const uint32_t *r = records + (size_t)slots[w] * L.record_words;
    for (int p = lane; p < obs; p += 32) {
        S[(size_t)w * obs + p] = __uint_as_float(r[L.off_state + p]);
        S2[(size_t)w * obs + p] = __uint_as_float(r[L.off_next_state + p]);
    }
    const uint8_t *id8 = reinterpret_cast<const uint8_t *>(r + L.off_avail);
    for (int k = lane; k < A; k += 32) ids[(size_t)w * A + k] = dynamic ? (int)id8[k] : k;
    if (lane == 0) {
        const uint32_t fl = r[L.off_flags];
        act[w] = (int)r[L.off_action];
        R[w] = __uint_as_float(r[L.off_reward]);
        T[w] = (fl & 1u) ? 1.f : 0.f;
        cnt[w] = dynamic ? min((int)((fl >> 8) & 0xffffu), A) : A;
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
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
        if (ov > best || (ov == best && ok < bk)) { best = ov; bk = ok; }
    }
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
struct prl_qrdqn {
    prl_qrdqn_cfg cfg;
    int P;
    int W1, b1, W2, b2, W3, b3;
    float *q, *q_m, *q_v, *q_x, *q_t;
    int64_t adam_step;
    // workspace
    float *S, *S2, *R, *T, *P1, *h1, *h2, *theta, *P1t, *c1t, *c2t, *qt, *tq, *dtheta, *rowabs, *dh2, *dh1, *grad;
    int *act, *cnt, *ids;
    int32_t *slots, *logical;
    float2 *scal;
    int *target_on;
    QrCall *call;
    int *round_idx;
    size_t tail_bytes;
    bool use_graph;
    cudaGraphExec_t graph_exec[2];            // [0] rounds from a replay buffer, [1] learn_batch on a dense batch
    int graph_batch[2];
    const uint32_t *graph_buf;
    int graph_dynamic;
    int launches_per_round;
    char *tail_host[2];
    cudaEvent_t tail_done[2];
    int tail_next;
    int64_t last_launches;
};

static int64_t al64(int64_t x) { return (x + 255) / 256 * 256; }

// per-call tail of the workspace: scal float2[MR] | target_on int32[MR] | call (8-byte aligned) | round_idx
static size_t qr_call_offset(int MR) { return ((size_t)MR * 12 + 7) / 8 * 8; }
static size_t qr_tail_bytes(int MR) { return qr_call_offset(MR) + sizeof(QrCall) + 4; }

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

struct QrWs { int64_t off[32]; int64_t total; };
static QrWs qr_ws(const prl_qrdqn_cfg *c, int P) {
    QrWs w; int64_t o = 0; int k = 0;
    const int64_t B = c->max_batch, O = c->obs_dim, A = c->n_actions, N = c->num_quantiles, BA = B * A;
    const int64_t H1 = c->hidden1, H2 = c->hidden2;
    auto add = [&](int64_t words) { w.off[k++] = o; o = al64(o + words * 4); };
    add(B * O); add(B * O); add(B); add(B);                                   // S S2 R T
    add(B * H1); add(B * H1); add(B * H2); add(B * N);                        // P1 h1 h2 theta      (online, taken action)
    add(B * H1); add(BA * H1); add(BA * H2); add(BA * N);                     // P1t c1t c2t qt      (target, every slot)
    add(B * N); add(B * N); add(B);                                           // tq dtheta rowabs
    add(B * H2); add(B * H1); add(P);                                         // dh2 dh1 grad
    add(B); add(B); add(BA);                                                  // act cnt ids (int32)
    add((int64_t)c->max_rounds * B); add((int64_t)c->max_rounds * B);        // slots logical (int32)
    add(((int64_t)qr_tail_bytes(c->max_rounds) + 3) / 4);                     // scal | target_on | call | round_idx
    w.total = o;
    return w;
}
extern "C" int64_t prl_qrdqn_workspace_bytes(const prl_qrdqn_cfg *c) {
    if (qr_check(c)) return -1;
    prl_qrdqn t; t.cfg = *c; qr_layout(&t);
    return qr_ws(c, t.P).total;
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
    QrWs w = qr_ws(cfg, s->P);
    char *b = (char *)workspace;
    float **f[] = {&s->S, &s->S2, &s->R, &s->T, &s->P1, &s->h1, &s->h2, &s->theta, &s->P1t, &s->c1t, &s->c2t, &s->qt, &s->tq, &s->dtheta,
                   &s->rowabs, &s->dh2, &s->dh1, &s->grad};
    int k = 0;
    for (auto p : f) *p = (float *)(b + w.off[k++]);
    s->act = (int *)(b + w.off[k++]); s->cnt = (int *)(b + w.off[k++]); s->ids = (int *)(b + w.off[k++]);
    s->slots = (int32_t *)(b + w.off[k++]); s->logical = (int32_t *)(b + w.off[k++]);
    char *tail = b + w.off[k++];
    const int MR = cfg->max_rounds;
    s->scal = (float2 *)tail;
    s->target_on = (int *)(tail + (size_t)MR * 8);
    s->call = (QrCall *)(tail + qr_call_offset(MR));
    s->round_idx = (int *)(s->call + 1);
    s->tail_bytes = qr_tail_bytes(MR);
    s->tail_next = 0; s->use_graph = true; s->graph_exec[0] = s->graph_exec[1] = nullptr; s->graph_batch[0] = s->graph_batch[1] = 0;
    s->graph_buf = nullptr; s->graph_dynamic = -1; s->last_launches = 0; s->launches_per_round = 0;
    cudaError_t e = cudaSuccess;
    int made = 0;   // pinned buffer / event pairs fully created
    s->tail_host[0] = s->tail_host[1] = nullptr;
    for (int i = 0; i < 2 && e == cudaSuccess; i++) {
        e = cudaHostAlloc((void **)&s->tail_host[i], s->tail_bytes, cudaHostAllocDefault);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->tail_done[i], cudaEventDisableTiming);
        if (e == cudaSuccess) made++;
    }
    if (e != cudaSuccess) {
        for (int i = 0; i < made; i++) { cudaEventDestroy(s->tail_done[i]); cudaFreeHost(s->tail_host[i]); }
        if (made < 2 && s->tail_host[made]) cudaFreeHost(s->tail_host[made]);   // its event was not created
        delete s;
        return fail(PRL_ECUDA, "prl_qrdqn_create: %s", cudaGetErrorString(e));
    }
    *out = s;
    return PRL_OK;
}
extern "C" int prl_qrdqn_destroy(prl_qrdqn *s) {
    if (!s) return PRL_OK;
    for (int i = 0; i < 2; i++) { cudaEventSynchronize(s->tail_done[i]); cudaEventDestroy(s->tail_done[i]); cudaFreeHost(s->tail_host[i]); }
    for (int i = 0; i < 2; i++) if (s->graph_exec[i]) cudaGraphExecDestroy(s->graph_exec[i]);
    delete s;
    return PRL_OK;
}
extern "C" int64_t prl_qrdqn_adam_step(const prl_qrdqn *s) { return s ? s->adam_step : -1; }

extern "C" int prl_qrdqn_set_lr(prl_qrdqn *s, double lr) {
    PRL_REQUIRE(s, "null handle");
    PRL_REQUIRE(lr >= 0.0, "the learning rate must be non-negative");
    s->cfg.lr = lr;
    return PRL_OK;
}

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
static int qr_round(prl_qrdqn *s, prl_buf *buf, int B, cudaStream_t st) {
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

// per-call block (Adam scalars of every round as torch evaluates them in double, target-update flags, decay, beta,
// pointers), uploaded on `st`.  steps0 = the training-step count the reference's learn_batch sees in round 0; round r
// updates the target when (steps0 + r + 1) % target_update_freq == 0.
static int qr_upload(prl_qrdqn *s, int rounds, int64_t steps0, double beta, float *out_loss, const QrCall &dense, cudaStream_t st) {
    const prl_qrdqn_cfg &c = s->cfg;
    const int sb = s->tail_next; s->tail_next ^= 1;
    PRL_CUDA(cudaEventSynchronize(s->tail_done[sb]));
    char *tail = s->tail_host[sb];
    const int MR = c.max_rounds;
    float2 *hs = reinterpret_cast<float2 *>(tail);
    int *on = reinterpret_cast<int *>(tail + (size_t)MR * 8);
    for (int r = 0; r < rounds; r++) {
        const double step = (double)(s->adam_step + r + 1);
        const double bc1 = 1.0 - pow(c.beta1, step), bc2 = 1.0 - pow(c.beta2, step);
        hs[r] = make_float2((float)(c.lr / bc1), (float)sqrt(bc2));
        on[r] = (steps0 + r + 1) % c.target_update_freq == 0 ? 1 : 0;
    }
    QrCall *hc = reinterpret_cast<QrCall *>(tail + qr_call_offset(MR));
    *hc = dense;
    hc->slots = s->slots; hc->out_loss = out_loss;
    hc->decay = (float)(1.0 - c.lr * c.weight_decay);
    hc->beta = (float)beta;
    *reinterpret_cast<int *>(hc + 1) = 0;
    PRL_CUDA(cudaMemcpyAsync(s->scal, tail, s->tail_bytes, cudaMemcpyHostToDevice, st));
    PRL_CUDA(cudaEventRecord(s->tail_done[sb], st));
    return PRL_OK;
}

static int qr_run(prl_qrdqn *s, prl_buf *buf, int rounds, int batch, cudaStream_t st) {
    const int g = buf ? 0 : 1;
    const int dynamic = (buf && (buf->desc.flags & PRL_BUF_DYNAMIC_ACTIONS)) ? 1 : 0;
    if (s->use_graph) {
        if (!s->graph_exec[g] || s->graph_batch[g] != batch || (buf && (s->graph_buf != buf->records || s->graph_dynamic != dynamic))) {
            if (s->graph_exec[g]) { cudaGraphExecDestroy(s->graph_exec[g]); s->graph_exec[g] = nullptr; }
            cudaStream_t cs;
            PRL_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
            cudaGraph_t graph = nullptr;
            cudaError_t e = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
            if (e == cudaSuccess) {
                qr_round(s, buf, batch, cs);
                e = cudaStreamEndCapture(cs, &graph);
            }
            if (e == cudaSuccess) e = cudaGraphInstantiate(&s->graph_exec[g], graph, 0);
            if (graph) cudaGraphDestroy(graph);
            cudaStreamDestroy(cs);
            if (e != cudaSuccess) { s->graph_exec[g] = nullptr; return fail(PRL_ECUDA, "prl_qrdqn: graph capture failed: %s", cudaGetErrorString(e)); }
            s->graph_batch[g] = batch;
            if (buf) { s->graph_buf = buf->records; s->graph_dynamic = dynamic; }
        }
        for (int r = 0; r < rounds; r++) PRL_CUDA(cudaGraphLaunch(s->graph_exec[g], st));
    } else {
        for (int r = 0; r < rounds; r++) {
            int rc = qr_round(s, buf, batch, st);
            if (rc) return rc;
        }
    }
    PRL_CUDA(cudaGetLastError());
    s->adam_step += rounds;
    s->last_launches = (int64_t)s->launches_per_round * rounds;
    return PRL_OK;
}

extern "C" int prl_qrdqn_learn(prl_qrdqn *s, prl_buf *buf, int rounds, int batch, int64_t training_steps, double beta, float *out_loss,
                               int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && out_loss, "null argument");
    const prl_qrdqn_cfg &c = s->cfg;
    PRL_REQUIRE(rounds > 0 && rounds <= c.max_rounds && batch > 0 && batch <= c.max_batch, "rounds / batch outside the configured maxima");
    PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.obs_dim == c.obs_dim && buf->desc.n_actions == c.n_actions,
                "QR-DQN needs a discrete-action buffer with obs_dim = %d and n_actions = %d", c.obs_dim, c.n_actions);
    PRL_REQUIRE(buf->shard_world <= 1, "the buffer is one shard of a multi-GPU buffer: QR-DQN samples local buffers only");
    cudaStream_t st = (cudaStream_t)stream_;
    int rc = prl_buf_sample_indices(buf, rounds, batch, out_logical ? out_logical : s->logical, s->slots, stream_);
    if (rc) return rc;
    QrCall dense;
    memset(&dense, 0, sizeof(dense));
    rc = qr_upload(s, rounds, training_steps + 1, beta, out_loss, dense, st);   // PolicyLearner.learn counts the round first
    if (rc) return rc;
    return qr_run(s, buf, rounds, batch, st);
}

extern "C" int prl_qrdqn_learn_batch(prl_qrdqn *s, int batch, const float *state, const int32_t *action_id, const float *reward,
                                     const float *next_state, const uint8_t *terminated, const int32_t *next_ids,
                                     const int32_t *next_count, int64_t training_steps, double beta, float *out_loss, void *stream_) {
    PRL_REQUIRE(s && state && action_id && reward && next_state && terminated && out_loss, "null argument");
    PRL_REQUIRE(batch > 0 && batch <= s->cfg.max_batch, "batch outside the configured maximum");
    cudaStream_t st = (cudaStream_t)stream_;
    QrCall dense;
    memset(&dense, 0, sizeof(dense));
    dense.d_state = state; dense.d_next_state = next_state; dense.d_reward = reward; dense.d_action_id = action_id;
    dense.d_next_ids = next_ids; dense.d_next_cnt = next_count; dense.d_term = terminated;
    int rc = qr_upload(s, 1, training_steps, beta, out_loss, dense, st);
    if (rc) return rc;
    return qr_run(s, nullptr, 1, batch, st);
}

extern "C" int prl_qrdqn_set_graph(prl_qrdqn *s, int enable) {
    PRL_REQUIRE(s, "null handle");
    s->use_graph = enable != 0;
    return PRL_OK;
}
extern "C" int64_t prl_qrdqn_last_launches(const prl_qrdqn *s) { return s ? s->last_launches : -1; }
