// cql.cu — conservative DQN / DoubleDQN (DeepQLearning / DoubleDQN built with is_conservative=True: CQL), driven by
// PolicyLearner.learn or called directly on a caller's batch (offline_learning / PearlAgent.learn_batch), replacing
//   policy_learners/sequential_decision_making/deep_td_learning.py   forward, loss, learn_batch (target update FIRST,
//       MSE Bellman loss + alpha * CQL term, AdamW step, reported mean |q - y|)
//   policy_learners/sequential_decision_making/deep_q_learning.py    get_next_state_values (max over available slots)
//   policy_learners/sequential_decision_making/double_dqn.py         get_next_state_values (online first argmax, target value)
//   utils/functional_utils/learning/loss_fn_utils.py                 compute_cql_loss
//   neural_networks/sequential_decision_making/q_value_networks.py   VanillaQValueNetwork (state || one-hot action -> 1)
//
// One round: the soft target update in flagged rounds (with the CURRENT online parameters, before anything else), the
// online net over B*(A+1) rows (the A current-action slots c_b[k] and, as slot A, the taken action), the target net (and,
// for DoubleDQN, the online net) over the B*A next slots, the Bellman target, the MSE gradient on slot A, the CQL gradient
// on slots 0..A-1, the backward pass over B*(A+1) rows and AdamW(amsgrad).  Fixed launch sequence, captured once per
// (batch, buffer) into a CUDA graph and replayed (DESIGN.md §3.4).  alpha, the AdamW step sizes, the decay factor and the
// per-round target-update flags are read through the per-call block, so neither prl_cql_set_lr nor a new alpha needs a
// new capture.  fp32, fixed summation order, no float atomics: bit-reproducible run to run.
//
// The reference's CQL term, reproduced as it computes it:
//   cql = mean_b logsumexp_k Q(s_b, c_b[k]) - mean(Q_all.gather(1, one_hot(a_b)))
// batch.action is already one-hot when compute_cql_loss gathers with it, so the second term picks column 0 in A-1 places
// and column 1 in one place of every row: (1 / (B A)) sum_b [(A-1) Q(s_b, c_b[0]) + Q(s_b, c_b[1])].  Padded current slots
// (action id 0, unavailable-mask ignored) take part in both terms.  Hence, on the all-slot values,
//   d(alpha cql)/dQ(s_b, c_b[k]) = alpha (softmax_k / B - [k = 0] (A-1) / (B A) - [k = 1] / (B A)),     A >= 2.
#include <limits.h>
#include <math.h>

#include "common.cuh"
#include "rounds.cuh"
#include "gemm.cuh"
#include "qrows.cuh"

using namespace prl;

namespace {

constexpr int kMaxA = 255;   // next-action ids are stored as bytes

// per-call block the captured round reads through
struct CqlCall : QSetCall {
    const int32_t *d_curr_ids;                // [B][A] current slot ids; null: every action (slot k holds k)
    float alpha;                              // conservative_alpha
};

// rows of one round (load_row), and the A + 1 online slots of the row: cids[b][k] = c_b[k] for k < A, cids[b][A] = the
// taken action.  The ring stores no current action sets: every action, as B200ReplayBuffer.sample reports.
__global__ void __launch_bounds__(256, 8) k_cql_load(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int A, int dynamic,
                           const CqlCall *__restrict__ call, const int *__restrict__ round_idx, int B, float *__restrict__ S,
                           float *__restrict__ S2, float *__restrict__ R, float *__restrict__ T, int *__restrict__ cnt,
                           int *__restrict__ ids, int *__restrict__ cids) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    const QRow row = load_row<true>(records, L, obs, A, dynamic, call, round_idx, B, w, lane, S, S2, R, T, ids);
    int *crow = cids + (size_t)w * (A + 1);
    const int32_t *cid = records ? nullptr : call->d_curr_ids;
    for (int k = lane; k < A; k += 32) crow[k] = cid ? cid[(size_t)w * A + k] : k;
    if (lane == 0) {
        crow[A] = row.action;
        cnt[w] = row.cnt;
    }
}

// Bellman target, loss gradients and |q - y|.  One warp per row b; lane l handles slots l, l + 32, ...
//   DQN:        V = max over available next slots of Q'(s', .)
//   DoubleDQN:  g = first argmax over available next slots of Q(s', .), V = Q'(s', g)
//   y = V * gamma * (1 - terminated) + r;  dq[b][A] = fl(2 / B) (q - y)  (MSELoss)
//   dq[b][k] = alpha (softmax_k(Q(s_b, c_b[.])) / B - n_k / (B A)),  n_0 = A - 1, n_1 = 1, n_k = 0 otherwise
// q_all: [B][A + 1] online values (slot A = taken action); qt / qn: [B][A] target / online values at the next slots.
__global__ void __launch_bounds__(128) k_cql_target(int B, int A, int dbl, const float *__restrict__ q_all, const float *__restrict__ qt,
                                                    const float *__restrict__ qn, const int *__restrict__ cnt,
                                                    const float *__restrict__ term, const float *__restrict__ rew,
                                                    const CqlCall *__restrict__ call, float gamma, float *__restrict__ dq,
                                                    float *__restrict__ rowabs) {
    const int lane = threadIdx.x & 31, b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= B) return;
    const int n_ok = cnt[b];
    const float *sel = (dbl ? qn : qt) + (size_t)b * A;
    float best = -INFINITY;
    int bk = INT_MAX;
    for (int k = lane; k < A; k += 32) {
        const float v = k < n_ok ? sel[k] : -INFINITY;
        if (v > best || (v == best && k < bk)) { best = v; bk = k; }
    }
    warp_first_max(best, bk);
    const float V = dbl ? qt[(size_t)b * A + (bk == INT_MAX ? 0 : bk)] : best;
    const float *l = q_all + (size_t)b * (A + 1);
    float *d = dq + (size_t)b * (A + 1);
    cql_slot_grad(A, B, call->alpha, lane, [&](int k) { return l[k]; }, [&](int k, float g) { d[k] = g; });
    if (lane == 0) {
        const float y = __fadd_rn(__fmul_rn(__fmul_rn(V, gamma), __fsub_rn(1.f, term[b])), rew[b]);
        const float e = __fsub_rn(l[A], y);
        d[A] = __fmul_rn(__fdiv_rn(2.f, (float)B), e);
        rowabs[b] = fabsf(e);
    }
}

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_cql : FlatQ<prl_cql, CqlCall, prl_cql_cfg> {
    static constexpr const char *kFn = "prl_cql", *kName = "CQL";
    static constexpr int kGraphs = 3;
    int W1, b1, W2, b2, W3, b3;
    // workspace
    float *S, *S2, *R, *T, *P1, *c1, *c2, *qa, *P1t, *c1t, *c2t, *qt, *qn, *dq, *rowabs, *dc2, *dc1, *dh1, *grad;
    int *cnt, *ids, *cids;
    static int check(const prl_cql_cfg *c);
    static void layout(prl_cql *s);
    static int64_t carve(prl_cql *s, void *base);
    static int round(prl_cql *s, prl_buf *buf, int B, cudaStream_t st);
};

void prl_cql::layout(prl_cql *s) {
    const prl_cql_cfg &c = s->cfg;
    const int D = c.obs_dim + c.n_actions;
    int o = 0;
    s->W1 = o; o += c.hidden1 * D; s->b1 = o; o += c.hidden1;
    s->W2 = o; o += c.hidden2 * c.hidden1; s->b2 = o; o += c.hidden2;
    s->W3 = o; o += c.hidden2; s->b3 = o; o += 1;
    s->P = o;
}

int prl_cql::check(const prl_cql_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->hidden1 > 0 && c->hidden2 > 0, "dimensions must be positive");
    PRL_REQUIRE(c->n_actions >= 2 && c->n_actions <= kMaxA,
                "n_actions must be in [2, %d]: the reference's CQL term gathers column 1 of the current-action values", kMaxA);
    PRL_REQUIRE(c->target_update_freq > 0, "target_update_freq must be positive");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    // the online pass over B (A + 1) slot rows indexes its activations (and the tensor-core operand rows) with 32-bit ints
    const int64_t slot_elems = (int64_t)c->max_batch * (c->n_actions + 1) * (c->hidden1 > c->hidden2 ? c->hidden1 : c->hidden2);
    PRL_REQUIRE(slot_elems < ((int64_t)1 << 31),
                "max_batch * (n_actions + 1) * max(hidden1, hidden2) = %lld must stay below 2^31 (32-bit element offsets)",
                (long long)slot_elems);
    return PRL_OK;
}

// the workspace, in order; base == null: only its size
int64_t prl_cql::carve(prl_cql *s, void *base) {
    const prl_cql_cfg &c = s->cfg;
    const int64_t B = c.max_batch, O = c.obs_dim, A = c.n_actions, BA = B * A, BA1 = B * (A + 1), H1 = c.hidden1, H2 = c.hidden2;
    Carve w{(char *)base};
    w(s->S, B * O); w(s->S2, B * O); w(s->R, B); w(s->T, B);
    w(s->P1, B * H1); w(s->c1, BA1 * H1); w(s->c2, BA1 * H2); w(s->qa, BA1);                 // online, A + 1 slots per row
    w(s->P1t, B * H1); w(s->c1t, BA * H1); w(s->c2t, BA * H2); w(s->qt, BA); w(s->qn, BA);   // next slots
    w(s->dq, BA1); w(s->rowabs, B);
    w(s->dc2, BA1 * H2); w(s->dc1, BA1 * H1); w(s->dh1, B * H1); w(s->grad, s->P);
    w(s->cnt, B); w(s->ids, BA); w(s->cids, BA1);
    s->carve_tail(w, c.max_rounds, B);
    return w.bytes;
}

extern "C" int64_t prl_cql_param_count(const prl_cql_cfg *c) { return prl_cql::param_count(c); }
extern "C" int64_t prl_cql_workspace_bytes(const prl_cql_cfg *c) { return prl_cql::workspace_bytes(c); }
extern "C" int prl_cql_create(prl_cql **out, const prl_cql_cfg *cfg, float *w, float *w_target, float *exp_avg, float *exp_avg_sq,
                              float *max_exp_avg_sq, int64_t adam_step, void *workspace) {
    return prl_cql::create(out, cfg, w, w_target, exp_avg, exp_avg_sq, max_exp_avg_sq, adam_step, workspace);
}
extern "C" int prl_cql_destroy(prl_cql *s) { return prl_cql::destroy(s); }
extern "C" int64_t prl_cql_adam_step(const prl_cql *s) { return prl_cql::adam_step_of(s); }
extern "C" int prl_cql_set_adam_step(prl_cql *s, int64_t step) { return prl_cql::set_adam_step(s, step); }
extern "C" int prl_cql_set_lr(prl_cql *s, double lr) { return prl_cql::set_lr(s, lr); }
extern "C" int prl_cql_set_graph(prl_cql *s, int enable) { return prl_cql::set_graph(s, enable); }
extern "C" int64_t prl_cql_last_launches(const prl_cql *s) { return prl_cql::last_launches_of(s); }

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
int prl_cql::round(prl_cql *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_cql_cfg &c = s->cfg;
    const int O = c.obs_dim, A = c.n_actions, D = O + A, H1 = c.hidden1, H2 = c.hidden2, BA = B * A, BA1 = B * (A + 1);
    // the decay factor is overridden by call->decay (k_adamw's decay pointer)
    const AdamHp h = adam_hp(0.0, c.beta1, c.beta2, c.eps, c.weight_decay);
    GemmLauncher L; L.st = st;
    const float *w = s->q, *t = s->q_t;
    float *g = s->grad;
    const int eb = 256;
    int small = 0;
    const int dynamic = (buf && (buf->desc.flags & PRL_BUF_DYNAMIC_ACTIONS)) ? 1 : 0;
    k_cql_load<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf ? buf->records : nullptr, buf ? buf->lay : prl_buf_layout{}, O, A, dynamic,
                                                     s->call, s->round_idx, B, s->S, s->S2, s->R, s->T, s->cnt, s->ids, s->cids);
    // ---------------- target update first, with the current online parameters (flagged rounds only)
    k_soft_update_flagged<<<(s->P + eb - 1) / eb, eb, 0, st>>>(s->P, s->q, s->q_t, (float)c.tau, (float)(1.0 - c.tau), s->target_on,
                                                               s->round_idx);
    small += 2;
    // ---------------- online net over the A current slots and the taken action (kept for the backward pass)
    L.fwd(mat(s->S, O), B, w + s->W1, D, 0, w + s->b1, 0, H1, O, false, s->P1, H1, 0);
    k_fold_expand<<<(unsigned)(((long long)BA1 * H1 + eb - 1) / eb), eb, 0, st>>>(B, A + 1, H1, s->P1, w + s->W1 + O, D, 0, s->cids, s->c1);
    L.fwd(mat(s->c1, H1), BA1, w + s->W2, H1, 0, w + s->b2, 0, H2, H1, true, s->c2, H2, 0);
    L.fwd(mat(s->c2, H2), BA1, w + s->W3, H2, 0, w + s->b3, 0, 1, H2, false, s->qa, 1, 0);
    small++;
    // ---------------- DoubleDQN: the online net over the next slots (greedy slot); then the target net over them
    auto next_pass = [&](const float *net, float *out) {
        L.fwd(mat(s->S2, O), B, net + s->W1, D, 0, net + s->b1, 0, H1, O, false, s->P1t, H1, 0);
        k_fold_expand<<<(unsigned)(((long long)BA * H1 + eb - 1) / eb), eb, 0, st>>>(B, A, H1, s->P1t, net + s->W1 + O, D, 0, s->ids, s->c1t);
        L.fwd(mat(s->c1t, H1), BA, net + s->W2, H1, 0, net + s->b2, 0, H2, H1, true, s->c2t, H2, 0);
        L.fwd(mat(s->c2t, H2), BA, net + s->W3, H2, 0, net + s->b3, 0, 1, H2, false, out, 1, 0);
        small++;
    };
    if (c.double_dqn) next_pass(w, s->qn);
    next_pass(t, s->qt);
    // ---------------- Bellman target, MSE gradient at the taken action, CQL gradient at the current slots
    k_cql_target<<<(B * 32 + 127) / 128, 128, 0, st>>>(B, A, c.double_dqn, s->qa, s->qt, s->qn, s->cnt, s->T, s->R, s->call, (float)c.gamma,
                                                      s->dq, s->rowabs);
    small++;
    // ---------------- backward through the online net over B*(A+1) rows
    L.bwd_w(s->dq, 1, 0, BA1, 1, mat(s->c2, H2), H2, g + s->W3, H2, 0, g + s->b3, 0);
    k_head_bwd<<<(unsigned)(((long long)BA1 * H2 + eb - 1) / eb), eb, 0, st>>>(BA1, H2, s->dq, w + s->W3, 0, s->c2, s->dc2);
    L.bwd_w(s->dc2, H2, 0, BA1, H2, mat(s->c1, H1), H1, g + s->W2, H1, 0, g + s->b2, 0);
    L.bwd_x(s->dc2, H2, 0, BA1, H2, w + s->W2, H1, 0, 0, H1, s->dc1, H1, 0, s->c1, H1, 0, false);
    k_slot_rowsum<<<(B * H1 + eb - 1) / eb, eb, 0, st>>>(B, A + 1, H1, s->dc1, s->dh1);
    L.bwd_w(s->dh1, H1, 0, B, H1, mat(s->S, O), O, g + s->W1, D, 0, g + s->b1, 0);                   // state columns + b1
    k_fold_w1a_grad<<<(H1 * A + eb - 1) / eb, eb, 0, st>>>(BA1, A, H1, s->cids, s->dc1, g + s->W1 + O, D, 0);
    small += 3;
    // ---------------- AdamW(amsgrad); the target was updated at the start of the round
    k_adamw<<<(s->P + eb - 1) / eb, eb, 0, st>>>(s->P, s->q, s->q_m, s->q_v, s->q_x, g, h, s->scal, s->round_idx, nullptr, 0.f, 0.f,
                                                &s->call->decay);
    k_round_report<<<1, 256, 0, st>>>(B, s->rowabs, s->call, s->round_idx);
    small += 2;
    s->launches_per_round = L.count + small;
    return PRL_OK;
}

extern "C" int prl_cql_learn(prl_cql *s, prl_buf *buf, int rounds, int batch, int64_t training_steps, double alpha, float *out_loss,
                             int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && out_loss, "null argument");
    CqlCall call{};
    call.alpha = (float)alpha; call.out_loss = out_loss;
    return prl_cql::learn(s, buf, rounds, batch, training_steps, out_logical, call, stream_);
}

extern "C" int prl_cql_learn_batch(prl_cql *s, int batch, const float *state, const int32_t *action_id, const float *reward,
                                   const float *next_state, const uint8_t *terminated, const int32_t *curr_ids,
                                   const int32_t *next_ids, const int32_t *next_count, int64_t training_steps, double alpha,
                                   float *out_loss, void *stream_) {
    PRL_REQUIRE(s && state && action_id && reward && next_state && terminated && out_loss, "null argument");
    CqlCall dense{};
    dense.d_state = state; dense.d_next_state = next_state; dense.d_reward = reward; dense.d_action_id = action_id;
    dense.d_curr_ids = curr_ids; dense.d_next_ids = next_ids; dense.d_next_cnt = next_count; dense.d_term = terminated;
    dense.alpha = (float)alpha;
    dense.out_loss = out_loss;
    return prl_cql::learn_batch(s, batch, training_steps, dense, stream_);
}

// Q(s, a) for every action: the online forward of the round on n rows (chunks of max_batch rows through the workspace)
extern "C" int prl_cql_q_values(prl_cql *s, int n, const float *state, int target, float *out_q, void *stream_) {
    PRL_REQUIRE(s && state && out_q, "null argument");
    if (n <= 0) return PRL_OK;
    const prl_cql_cfg &c = s->cfg;
    const int O = c.obs_dim, A = c.n_actions, D = O + A, H1 = c.hidden1, H2 = c.hidden2, eb = 256;
    const float *w = target ? s->q_t : s->q;
    GemmLauncher L; L.st = (cudaStream_t)stream_;
    for (int r0 = 0; r0 < n; r0 += c.max_batch) {
        const int m = n - r0 < c.max_batch ? n - r0 : c.max_batch, mA = m * A;
        L.fwd(mat(state + (size_t)r0 * O, O), m, w + s->W1, D, 0, w + s->b1, 0, H1, O, false, s->P1, H1, 0);
        k_fold_expand<<<(unsigned)(((long long)mA * H1 + eb - 1) / eb), eb, 0, L.st>>>(m, A, H1, s->P1, w + s->W1 + O, D, 0, nullptr, s->c1);
        L.fwd(mat(s->c1, H1), mA, w + s->W2, H1, 0, w + s->b2, 0, H2, H1, true, s->c2, H2, 0);
        L.fwd(mat(s->c2, H2), mA, w + s->W3, H2, 0, w + s->b3, 0, 1, H2, false, out_q + (size_t)r0 * A, 1, 0);
    }
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}
