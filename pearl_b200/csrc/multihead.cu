// multihead.cu — multi-head DQN / DoubleDQN (DeepQLearning / DoubleDQN built with VanillaQValueMultiHeadNetwork), plain
// or conservative (CQL), driven by PolicyLearner.learn or called directly on a caller's batch (PearlAgent.learn_batch /
// offline_learning), replacing
//   neural_networks/sequential_decision_making/q_value_networks.py   VanillaQValueMultiHeadNetwork (state -> one Q value
//       per action; get_q_values = bmm(one-hot slots, Q(s)), so a slot reads the head column of the id it holds)
//   policy_learners/sequential_decision_making/deep_td_learning.py   forward, loss, learn_batch (target update FIRST,
//       MSE Bellman loss [+ alpha * CQL term], AdamW step, reported mean |q - y|)
//   policy_learners/sequential_decision_making/deep_q_learning.py    get_next_state_values (max over available slots)
//   policy_learners/sequential_decision_making/double_dqn.py         get_next_state_values (online first argmax, target value)
//   utils/functional_utils/learning/loss_fn_utils.py                 compute_cql_loss
//
// One forward pass per state: the online net on the B states (for DoubleDQN stacked with the B next states into one
// 2B-row product), the target net on the B next states, then one warp per row for q, V', y, |q - y| and the head gradient
// row dQ[b][0..A), and the backward pass over B rows.  Round: the soft target update in flagged rounds (with the CURRENT
// online parameters, before anything else), the passes above and AdamW(amsgrad).  Fixed launch sequence, captured once per
// (batch, buffer) into a CUDA graph and replayed (DESIGN.md §3.4).  alpha, the AdamW step sizes, the decay factor and the
// per-round target-update flags are read through the per-call block, so neither prl_mhq_set_lr nor a new alpha needs a new
// capture.  fp32, fixed summation order, no float atomics: bit-reproducible run to run.
//
// Head gradient of row b (column j of dQ[b]):
//   [j = a_b] fl(2 / B) (q_b - y_b)                                     MSELoss on q_b = Q(s_b)[a_b]
//   + sum over current slots k with c_b[k] = j, k ascending, of
//     alpha (softmax_k / B - n_k / (B A)),  n_0 = A - 1, n_1 = 1        conservative only: the reference's CQL term as it
//                                                                       computes it (cql.cu), whose data part reads slot
//                                                                       columns 0 and 1; padded slots (id 0) repeat an id,
//                                                                       so their terms add on one head column
// the CQL terms summed first, the MSE term added last.
#include <limits.h>
#include <math.h>

#include "common.cuh"
#include "rounds.cuh"
#include "gemm.cuh"
#include "qrows.cuh"

using namespace prl;

namespace {

constexpr int kMaxA = 255;   // next-action ids are stored as bytes
constexpr int kColsPerLane = (kMaxA + 31) / 32;

// per-call block the captured round reads through
struct MhqCall : QSetCall {
    const int32_t *d_curr_ids;                // [B][A] current slot ids; null: every action (slot k holds k)
    float alpha;                              // conservative_alpha
};

// rows of one round (load_row): S holds the states, S2 the next states; the taken action and the current slot ids.  The
// ring stores no current action sets: every action, as B200ReplayBuffer.sample reports.
__global__ void __launch_bounds__(256, 8) k_mhq_load(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int A, int dynamic,
                           const MhqCall *__restrict__ call, const int *__restrict__ round_idx, int B, float *__restrict__ S,
                           float *__restrict__ S2, float *__restrict__ R, float *__restrict__ T, int *__restrict__ act,
                           int *__restrict__ cnt, int *__restrict__ ids, int *__restrict__ cur) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    const QRow row = load_row<true>(records, L, obs, A, dynamic, call, round_idx, B, w, lane, S, S2, R, T, ids);
    int *crow = cur + (size_t)w * A;
    const int32_t *cid = records ? nullptr : call->d_curr_ids;
    for (int k = lane; k < A; k += 32) crow[k] = cid ? cid[(size_t)w * A + k] : k;
    if (lane == 0) {
        act[w] = row.action;
        cnt[w] = row.cnt;
    }
}

// Bellman target, the head gradient row and |q - y|.  One warp per row b; lane l handles slots l, l + 32, ... and head
// columns l, l + 32, ...
//   DQN:        V = max over available next slots k of Q'(s')[id_k]
//   DoubleDQN:  k* = first argmax over available next slots of Q(s')[id_k], V = Q'(s')[id_k*]
//   y = V * gamma * (1 - terminated) + r;  q = Q(s)[a];  dQ[b][.] as in the file header
// qo: [B][A] online values at s; qn / qt: [B][A] online / target values at s'.
__global__ void __launch_bounds__(128) k_mhq_head(int B, int A, int dbl, int cons, const float *__restrict__ qo,
                                                  const float *__restrict__ qn, const float *__restrict__ qt,
                                                  const int *__restrict__ ids, const int *__restrict__ cnt,
                                                  const int *__restrict__ cur, const int *__restrict__ act,
                                                  const float *__restrict__ term, const float *__restrict__ rew,
                                                  const MhqCall *__restrict__ call, float gamma, float *__restrict__ dq,
                                                  float *__restrict__ rowabs) {
    __shared__ float sg[4][kMaxA + 1];
    __shared__ int sid[4][kMaxA + 1];
    const int lane = threadIdx.x & 31, wb = threadIdx.x >> 5, b = blockIdx.x * 4 + wb;
    if (b >= B) return;
    const int n_ok = cnt[b];
    const int *nid = ids + (size_t)b * A;
    const float *sel = (dbl ? qn : qt) + (size_t)b * A;
    float best = -INFINITY;
    int bk = INT_MAX;
    for (int k = lane; k < A; k += 32) {
        const float v = k < n_ok ? sel[nid[k]] : -INFINITY;
        if (v > best || (v == best && k < bk)) { best = v; bk = k; }
    }
    warp_first_max(best, bk);
    const float V = dbl ? qt[(size_t)b * A + nid[bk == INT_MAX ? 0 : bk]] : best;
    const float *l = qo + (size_t)b * A;
    const int a = act[b];
    const float y = __fadd_rn(__fmul_rn(__fmul_rn(V, gamma), __fsub_rn(1.f, term[b])), rew[b]);
    const float e = __fsub_rn(l[a], y);
    const float dqa = __fmul_rn(__fdiv_rn(2.f, (float)B), e);
    float acc[kColsPerLane];
#pragma unroll
    for (int c = 0; c < kColsPerLane; c++) acc[c] = 0.f;
    if (cons) {
        // the slot gradients are staged in shared memory and added per head column in ascending slot order
        const int *c_b = cur + (size_t)b * A;
        cql_slot_grad(A, B, call->alpha, lane, [&](int k) { return l[c_b[k]]; }, [&](int k, float g) {
            sg[wb][k] = g;
            sid[wb][k] = c_b[k];
        });
        __syncwarp();
        for (int k = 0; k < A; k++) {
            const int id = sid[wb][k];
            const float g = sg[wb][k];
#pragma unroll
            for (int c = 0; c < kColsPerLane; c++)
                if (id == lane + 32 * c) acc[c] = __fadd_rn(acc[c], g);
        }
    }
    float *d = dq + (size_t)b * A;
#pragma unroll
    for (int c = 0; c < kColsPerLane; c++) {
        const int j = lane + 32 * c;
        if (j < A) d[j] = j == a ? __fadd_rn(acc[c], dqa) : acc[c];
    }
    if (lane == 0) rowabs[b] = fabsf(e);
}

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_mhq : FlatQ<prl_mhq, MhqCall, prl_mhq_cfg> {
    static constexpr const char *kFn = "prl_mhq", *kName = "multi-head DQN";
    static constexpr int kGraphs = 3;
    int W1, b1, W2, b2, W3, b3;
    // workspace: S holds the states and, right after the round's B rows, the next states (one 2B-row online pass)
    float *S, *R, *T, *h1, *h2, *qo, *h1t, *h2t, *qt, *dq, *rowabs, *dh2, *dh1, *grad;
    int *act, *cnt, *ids, *cur;
    static int check(const prl_mhq_cfg *c);
    static int64_t layout(prl_mhq *s);
    static int64_t carve(prl_mhq *s, void *base);
    static int round(prl_mhq *s, prl_buf *buf, int B, cudaStream_t st);
};

// the parameter offsets and P, set when the count stays below 2^31; returns the count
int64_t prl_mhq::layout(prl_mhq *s) {
    const prl_mhq_cfg &c = s->cfg;
    int64_t o = 0, p[6];
    p[0] = o; o += (int64_t)c.hidden1 * c.obs_dim; p[1] = o; o += c.hidden1;
    p[2] = o; o += (int64_t)c.hidden2 * c.hidden1; p[3] = o; o += c.hidden2;
    p[4] = o; o += (int64_t)c.n_actions * c.hidden2; p[5] = o; o += c.n_actions;
    if (o < ((int64_t)1 << 31)) {
        s->W1 = (int)p[0]; s->b1 = (int)p[1]; s->W2 = (int)p[2]; s->b2 = (int)p[3]; s->W3 = (int)p[4]; s->b3 = (int)p[5];
        s->P = (int)o;
    }
    return o;
}

int prl_mhq::check(const prl_mhq_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->hidden1 > 0 && c->hidden2 > 0, "dimensions must be positive");
    PRL_REQUIRE(c->n_actions >= 1 && c->n_actions <= kMaxA, "n_actions must be in [1, %d]: next-action ids are stored as bytes", kMaxA);
    PRL_REQUIRE(!c->conservative || c->n_actions >= 2,
                "conservative updates need n_actions >= 2: the reference's CQL term gathers column 1 of the current-action values");
    PRL_REQUIRE(c->target_update_freq > 0, "target_update_freq must be positive");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    // the stacked online pass over 2 max_batch rows indexes its activations (and the tensor-core operand rows) with 32-bit ints
    int64_t wmax = c->obs_dim;
    for (int64_t x : {(int64_t)c->hidden1, (int64_t)c->hidden2, (int64_t)c->n_actions}) wmax = x > wmax ? x : wmax;
    const int64_t elems = 2 * (int64_t)c->max_batch * wmax;
    PRL_REQUIRE(elems < ((int64_t)1 << 31),
                "2 * max_batch * max(obs_dim, hidden1, hidden2, n_actions) = %lld must stay below 2^31 (32-bit element offsets)",
                (long long)elems);
    prl_mhq t; t.cfg = *c;
    const int64_t P = layout(&t);
    PRL_REQUIRE(P < ((int64_t)1 << 31), "the parameter count %lld must stay below 2^31 (32-bit element offsets)", (long long)P);
    return PRL_OK;
}

// the workspace, in order; base == null: only its size
int64_t prl_mhq::carve(prl_mhq *s, void *base) {
    const prl_mhq_cfg &c = s->cfg;
    const int64_t B = c.max_batch, B2 = 2 * B, O = c.obs_dim, A = c.n_actions, H1 = c.hidden1, H2 = c.hidden2;
    Carve w{(char *)base};
    w(s->S, B2 * O); w(s->R, B); w(s->T, B);
    w(s->h1, B2 * H1); w(s->h2, B2 * H2); w(s->qo, B2 * A);                 // online, states then next states
    w(s->h1t, B * H1); w(s->h2t, B * H2); w(s->qt, B * A);                  // target, next states
    w(s->dq, B * A); w(s->rowabs, B); w(s->dh2, B * H2); w(s->dh1, B * H1); w(s->grad, s->P);
    w(s->act, B); w(s->cnt, B); w(s->ids, B * A); w(s->cur, B * A);
    s->carve_tail(w, c.max_rounds, B);
    return w.bytes;
}

extern "C" int64_t prl_mhq_param_count(const prl_mhq_cfg *c) { return prl_mhq::param_count(c); }
extern "C" int64_t prl_mhq_workspace_bytes(const prl_mhq_cfg *c) { return prl_mhq::workspace_bytes(c); }
extern "C" int prl_mhq_create(prl_mhq **out, const prl_mhq_cfg *cfg, float *w, float *w_target, float *exp_avg, float *exp_avg_sq,
                              float *max_exp_avg_sq, int64_t adam_step, void *workspace) {
    return prl_mhq::create(out, cfg, w, w_target, exp_avg, exp_avg_sq, max_exp_avg_sq, adam_step, workspace);
}
extern "C" int prl_mhq_destroy(prl_mhq *s) { return prl_mhq::destroy(s); }
extern "C" int64_t prl_mhq_adam_step(const prl_mhq *s) { return prl_mhq::adam_step_of(s); }
extern "C" int prl_mhq_set_adam_step(prl_mhq *s, int64_t step) { return prl_mhq::set_adam_step(s, step); }
extern "C" int prl_mhq_set_lr(prl_mhq *s, double lr) { return prl_mhq::set_lr(s, lr); }
extern "C" int prl_mhq_set_graph(prl_mhq *s, int enable) { return prl_mhq::set_graph(s, enable); }
extern "C" int64_t prl_mhq_last_launches(const prl_mhq *s) { return prl_mhq::last_launches_of(s); }

// the net `net` on m rows X: layer activations into h1 / h2, the A head values into out
static void mhq_fwd(const prl_mhq *s, GemmLauncher &L, const float *net, const float *X, int m, float *h1, float *h2, float *out) {
    const prl_mhq_cfg &c = s->cfg;
    const int O = c.obs_dim, A = c.n_actions, H1 = c.hidden1, H2 = c.hidden2;
    L.fwd(mat(X, O), m, net + s->W1, O, 0, net + s->b1, 0, H1, O, true, h1, H1, 0);
    L.fwd(mat(h1, H1), m, net + s->W2, H1, 0, net + s->b2, 0, H2, H1, true, h2, H2, 0);
    L.fwd(mat(h2, H2), m, net + s->W3, H2, 0, net + s->b3, 0, A, H2, false, out, A, 0);
}

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
int prl_mhq::round(prl_mhq *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_mhq_cfg &c = s->cfg;
    const int O = c.obs_dim, A = c.n_actions, H1 = c.hidden1, H2 = c.hidden2;
    // the decay factor is overridden by call->decay (k_adamw's decay pointer)
    const AdamHp h = adam_hp(0.0, c.beta1, c.beta2, c.eps, c.weight_decay);
    GemmLauncher L; L.st = st;
    const float *w = s->q;
    float *g = s->grad, *S2 = s->S + (size_t)B * O;
    const int eb = 256;
    int small = 0;
    const int dynamic = (buf && (buf->desc.flags & PRL_BUF_DYNAMIC_ACTIONS)) ? 1 : 0;
    k_mhq_load<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf ? buf->records : nullptr, buf ? buf->lay : prl_buf_layout{}, O, A, dynamic,
                                                     s->call, s->round_idx, B, s->S, S2, s->R, s->T, s->act, s->cnt, s->ids, s->cur);
    // ---------------- target update first, with the current online parameters (flagged rounds only)
    k_soft_update_flagged<<<(s->P + eb - 1) / eb, eb, 0, st>>>(s->P, s->q, s->q_t, (float)c.tau, (float)(1.0 - c.tau), s->target_on,
                                                               s->round_idx);
    small += 2;
    // ---------------- online net on the states (kept for the backward pass) and, for DoubleDQN, the next states: rows
    // B..2B-1 of the same product; then the target net on the next states
    mhq_fwd(s, L, w, s->S, c.double_dqn ? 2 * B : B, s->h1, s->h2, s->qo);
    mhq_fwd(s, L, s->q_t, S2, B, s->h1t, s->h2t, s->qt);
    // ---------------- Bellman target and the head gradient rows
    k_mhq_head<<<(B + 3) / 4, 128, 0, st>>>(B, A, c.double_dqn, c.conservative, s->qo, s->qo + (size_t)B * A, s->qt, s->ids, s->cnt,
                                           s->cur, s->act, s->T, s->R, s->call, (float)c.gamma, s->dq, s->rowabs);
    small++;
    // ---------------- backward through the online net over the B state rows
    L.bwd_w(s->dq, A, 0, B, A, mat(s->h2, H2), H2, g + s->W3, H2, 0, g + s->b3, 0);
    L.bwd_x(s->dq, A, 0, B, A, w + s->W3, H2, 0, 0, H2, s->dh2, H2, 0, s->h2, H2, 0, false);
    L.bwd_w(s->dh2, H2, 0, B, H2, mat(s->h1, H1), H1, g + s->W2, H1, 0, g + s->b2, 0);
    L.bwd_x(s->dh2, H2, 0, B, H2, w + s->W2, H1, 0, 0, H1, s->dh1, H1, 0, s->h1, H1, 0, false);
    L.bwd_w(s->dh1, H1, 0, B, H1, mat(s->S, O), O, g + s->W1, O, 0, g + s->b1, 0);
    // ---------------- AdamW(amsgrad); the target was updated at the start of the round
    k_adamw<<<(s->P + eb - 1) / eb, eb, 0, st>>>(s->P, s->q, s->q_m, s->q_v, s->q_x, g, h, s->scal, s->round_idx, nullptr, 0.f, 0.f,
                                                &s->call->decay);
    k_round_report<<<1, 256, 0, st>>>(B, s->rowabs, s->call, s->round_idx);
    small += 2;
    s->launches_per_round = L.count + small;
    return PRL_OK;
}

extern "C" int prl_mhq_learn(prl_mhq *s, prl_buf *buf, int rounds, int batch, int64_t training_steps, double alpha, float *out_loss,
                             int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && out_loss, "null argument");
    MhqCall call{};
    call.alpha = (float)alpha; call.out_loss = out_loss;
    return prl_mhq::learn(s, buf, rounds, batch, training_steps, out_logical, call, stream_);
}

extern "C" int prl_mhq_learn_batch(prl_mhq *s, int batch, const float *state, const int32_t *action_id, const float *reward,
                                   const float *next_state, const uint8_t *terminated, const int32_t *curr_ids,
                                   const int32_t *next_ids, const int32_t *next_count, int64_t training_steps, double alpha,
                                   float *out_loss, void *stream_) {
    PRL_REQUIRE(s && state && action_id && reward && next_state && terminated && out_loss, "null argument");
    MhqCall dense{};
    dense.d_state = state; dense.d_next_state = next_state; dense.d_reward = reward; dense.d_action_id = action_id;
    dense.d_curr_ids = curr_ids; dense.d_next_ids = next_ids; dense.d_next_cnt = next_count; dense.d_term = terminated;
    dense.alpha = (float)alpha;
    dense.out_loss = out_loss;
    return prl_mhq::learn_batch(s, batch, training_steps, dense, stream_);
}

// Q(s)[a] for every action: the online (or target) forward of the round on n rows (chunks of max_batch rows through the
// workspace)
extern "C" int prl_mhq_q_values(prl_mhq *s, int n, const float *state, int target, float *out_q, void *stream_) {
    PRL_REQUIRE(s && state && out_q, "null argument");
    if (n <= 0) return PRL_OK;
    const prl_mhq_cfg &c = s->cfg;
    const float *w = target ? s->q_t : s->q;
    GemmLauncher L; L.st = (cudaStream_t)stream_;
    for (int r0 = 0; r0 < n; r0 += c.max_batch) {
        const int m = n - r0 < c.max_batch ? n - r0 : c.max_batch;
        mhq_fwd(s, L, w, state + (size_t)r0 * c.obs_dim, m, s->h1, s->h2, out_q + (size_t)r0 * c.n_actions);
    }
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}
