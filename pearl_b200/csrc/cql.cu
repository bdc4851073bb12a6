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

#include <new>

#include "common.cuh"
#include "gemm.cuh"

using namespace prl;

namespace {

constexpr int kMaxA = 255;   // next-action ids are stored as bytes

// per-call block the captured round reads through
struct CqlCall {
    const int32_t *slots;                     // [rounds][B] (learn)
    float *out_loss;                          // [rounds]
    // learn_batch: the caller's dense batch
    const float *d_state, *d_next_state, *d_reward;
    const int32_t *d_action_id;
    const int32_t *d_curr_ids;                // [B][A] current slot ids; null: every action (slot k holds k)
    const int32_t *d_next_ids, *d_next_cnt;   // may be null: every action available next
    const uint8_t *d_term;
    float decay;                              // AdamW decoupled decay 1 - lr * weight_decay
    float alpha;                              // conservative_alpha
};

// rows of one round: state, next state, reward, terminated, the next-action id of every slot with the available count, and
// the A + 1 online slots of the row: cids[b][k] = c_b[k] for k < A, cids[b][A] = the taken action.  records == null: pack
// the caller's dense batch.  The ring stores no current action sets: every action, as B200ReplayBuffer.sample reports.
__global__ void k_cql_load(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int A, int dynamic,
                           const CqlCall *__restrict__ call, const int *__restrict__ round_idx, int B, float *__restrict__ S,
                           float *__restrict__ S2, float *__restrict__ R, float *__restrict__ T, int *__restrict__ cnt,
                           int *__restrict__ ids, int *__restrict__ cids) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    int *crow = cids + (size_t)w * (A + 1);
    if (!records) {
        for (int p = lane; p < obs; p += 32) {
            S[(size_t)w * obs + p] = call->d_state[(size_t)w * obs + p];
            S2[(size_t)w * obs + p] = call->d_next_state[(size_t)w * obs + p];
        }
        const int32_t *nid = call->d_next_ids, *cid = call->d_curr_ids;
        for (int k = lane; k < A; k += 32) {
            ids[(size_t)w * A + k] = nid ? nid[(size_t)w * A + k] : k;
            crow[k] = cid ? cid[(size_t)w * A + k] : k;
        }
        if (lane == 0) {
            crow[A] = call->d_action_id[w];
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
    for (int k = lane; k < A; k += 32) {
        ids[(size_t)w * A + k] = dynamic ? (int)id8[k] : k;
        crow[k] = k;
    }
    if (lane == 0) {
        const uint32_t fl = r[L.off_flags];
        crow[A] = (int)r[L.off_action];
        R[w] = __uint_as_float(r[L.off_reward]);
        T[w] = (fl & 1u) ? 1.f : 0.f;
        cnt[w] = dynamic ? min((int)((fl >> 8) & 0xffffu), A) : A;
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
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
        if (ov > best || (ov == best && ok < bk)) { best = ov; bk = ok; }
    }
    const float V = dbl ? qt[(size_t)b * A + (bk == INT_MAX ? 0 : bk)] : best;
    const float *l = q_all + (size_t)b * (A + 1);
    // logsumexp over the A current slots: row max, then the sum of exp(l - max) (per lane in slot order, then a fixed tree)
    float mx = -INFINITY;
    for (int k = lane; k < A; k += 32) mx = fmaxf(mx, l[k]);
#pragma unroll
    for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float s = 0.f;
    for (int k = lane; k < A; k += 32) s += expf(l[k] - mx);
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float alpha = call->alpha, fB = (float)B, inv_ba = 1.f / ((float)B * (float)A);
    float *d = dq + (size_t)b * (A + 1);
    for (int k = lane; k < A; k += 32) {
        const float p = expf(l[k] - mx) / s;
        const float n_k = k == 0 ? (float)(A - 1) : (k == 1 ? 1.f : 0.f);
        d[k] = __fmul_rn(alpha, __fsub_rn(__fdiv_rn(p, fB), __fmul_rn(n_k, inv_ba)));
    }
    if (lane == 0) {
        const float y = __fadd_rn(__fmul_rn(__fmul_rn(V, gamma), __fsub_rn(1.f, term[b])), rew[b]);
        const float e = __fsub_rn(l[A], y);
        d[A] = __fmul_rn(__fdiv_rn(2.f, fB), e);
        rowabs[b] = fabsf(e);
    }
}

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_cql {
    prl_cql_cfg cfg;
    int P;
    int W1, b1, W2, b2, W3, b3;
    float *q, *q_t, *q_m, *q_v, *q_x;
    int64_t adam_step;
    // workspace
    float *S, *S2, *R, *T, *P1, *c1, *c2, *qa, *P1t, *c1t, *c2t, *qt, *qn, *dq, *rowabs, *dc2, *dc1, *dh1, *grad;
    int *cnt, *ids, *cids;
    int32_t *slots, *logical;
    float2 *scal;
    int *target_on;
    CqlCall *call;
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
static size_t cql_call_offset(int MR) { return ((size_t)MR * 12 + 7) / 8 * 8; }
static size_t cql_tail_bytes(int MR) { return cql_call_offset(MR) + sizeof(CqlCall) + 4; }

static void cql_layout(prl_cql *s) {
    const prl_cql_cfg &c = s->cfg;
    const int D = c.obs_dim + c.n_actions;
    int o = 0;
    s->W1 = o; o += c.hidden1 * D; s->b1 = o; o += c.hidden1;
    s->W2 = o; o += c.hidden2 * c.hidden1; s->b2 = o; o += c.hidden2;
    s->W3 = o; o += c.hidden2; s->b3 = o; o += 1;
    s->P = o;
}

static int cql_check(const prl_cql_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->hidden1 > 0 && c->hidden2 > 0, "dimensions must be positive");
    PRL_REQUIRE(c->n_actions >= 2 && c->n_actions <= kMaxA,
                "n_actions must be in [2, %d]: the reference's CQL term gathers column 1 of the current-action values", kMaxA);
    PRL_REQUIRE(c->target_update_freq > 0, "target_update_freq must be positive");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    return PRL_OK;
}

extern "C" int64_t prl_cql_param_count(const prl_cql_cfg *c) {
    if (cql_check(c)) return -1;
    prl_cql t; t.cfg = *c; cql_layout(&t);
    return t.P;
}

struct CqlWs { int64_t off[32]; int64_t total; };
static CqlWs cql_ws(const prl_cql_cfg *c, int P) {
    CqlWs w; int64_t o = 0; int k = 0;
    const int64_t B = c->max_batch, O = c->obs_dim, A = c->n_actions, BA = B * A, BA1 = B * (A + 1);
    const int64_t H1 = c->hidden1, H2 = c->hidden2;
    auto add = [&](int64_t words) { w.off[k++] = o; o = al64(o + words * 4); };
    add(B * O); add(B * O); add(B); add(B);                                   // S S2 R T
    add(B * H1); add(BA1 * H1); add(BA1 * H2); add(BA1);                      // P1 c1 c2 qa     (online, A + 1 slots per row)
    add(B * H1); add(BA * H1); add(BA * H2); add(BA); add(BA);                // P1t c1t c2t qt qn (next slots)
    add(BA1); add(B);                                                         // dq rowabs
    add(BA1 * H2); add(BA1 * H1); add(B * H1); add(P);                        // dc2 dc1 dh1 grad
    add(B); add(BA); add(BA1);                                                // cnt ids cids (int32)
    add((int64_t)c->max_rounds * B); add((int64_t)c->max_rounds * B);        // slots logical (int32)
    add(((int64_t)cql_tail_bytes(c->max_rounds) + 3) / 4);                    // scal | target_on | call | round_idx
    w.total = o;
    return w;
}
extern "C" int64_t prl_cql_workspace_bytes(const prl_cql_cfg *c) {
    if (cql_check(c)) return -1;
    prl_cql t; t.cfg = *c; cql_layout(&t);
    return cql_ws(c, t.P).total;
}

extern "C" int prl_cql_create(prl_cql **out, const prl_cql_cfg *cfg, float *w, float *w_target, float *exp_avg, float *exp_avg_sq,
                              float *max_exp_avg_sq, int64_t adam_step, void *workspace) {
    PRL_REQUIRE(out && w && w_target && exp_avg && exp_avg_sq && max_exp_avg_sq && workspace, "null argument");
    int rc = cql_check(cfg);
    if (rc) return rc;
    prl_cql *s = new (std::nothrow) prl_cql();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    cql_layout(s);
    s->q = w; s->q_t = w_target; s->q_m = exp_avg; s->q_v = exp_avg_sq; s->q_x = max_exp_avg_sq;
    s->adam_step = adam_step;
    CqlWs ws = cql_ws(cfg, s->P);
    char *b = (char *)workspace;
    float **f[] = {&s->S, &s->S2, &s->R, &s->T, &s->P1, &s->c1, &s->c2, &s->qa, &s->P1t, &s->c1t, &s->c2t, &s->qt, &s->qn,
                   &s->dq, &s->rowabs, &s->dc2, &s->dc1, &s->dh1, &s->grad};
    int k = 0;
    for (auto p : f) *p = (float *)(b + ws.off[k++]);
    s->cnt = (int *)(b + ws.off[k++]); s->ids = (int *)(b + ws.off[k++]); s->cids = (int *)(b + ws.off[k++]);
    s->slots = (int32_t *)(b + ws.off[k++]); s->logical = (int32_t *)(b + ws.off[k++]);
    char *tail = b + ws.off[k++];
    const int MR = cfg->max_rounds;
    s->scal = (float2 *)tail;
    s->target_on = (int *)(tail + (size_t)MR * 8);
    s->call = (CqlCall *)(tail + cql_call_offset(MR));
    s->round_idx = (int *)(s->call + 1);
    s->tail_bytes = cql_tail_bytes(MR);
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
        return fail(PRL_ECUDA, "prl_cql_create: %s", cudaGetErrorString(e));
    }
    *out = s;
    return PRL_OK;
}
extern "C" int prl_cql_destroy(prl_cql *s) {
    if (!s) return PRL_OK;
    for (int i = 0; i < 2; i++) { cudaEventSynchronize(s->tail_done[i]); cudaEventDestroy(s->tail_done[i]); cudaFreeHost(s->tail_host[i]); }
    for (int i = 0; i < 2; i++) if (s->graph_exec[i]) cudaGraphExecDestroy(s->graph_exec[i]);
    delete s;
    return PRL_OK;
}
extern "C" int64_t prl_cql_adam_step(const prl_cql *s) { return s ? s->adam_step : -1; }
extern "C" int prl_cql_set_adam_step(prl_cql *s, int64_t step) {
    PRL_REQUIRE(s, "null handle");
    PRL_REQUIRE(step >= 0, "the AdamW step count must be non-negative");
    s->adam_step = step;
    return PRL_OK;
}

extern "C" int prl_cql_set_lr(prl_cql *s, double lr) {
    PRL_REQUIRE(s, "null handle");
    PRL_REQUIRE(lr >= 0.0, "the learning rate must be non-negative");
    s->cfg.lr = lr;
    return PRL_OK;
}

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
static int cql_round(prl_cql *s, prl_buf *buf, int B, cudaStream_t st) {
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
    k_head_bwd<<<(BA1 * H2 + eb - 1) / eb, eb, 0, st>>>(BA1, H2, s->dq, w + s->W3, 0, s->c2, s->dc2);
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

// per-call block (Adam scalars of every round as torch evaluates them in double, target-update flags, decay, alpha,
// pointers), uploaded on `st`.  steps0 = the training-step count the reference's learn_batch sees in round 0; round r
// updates the target first when (steps0 + r + 1) % target_update_freq == 0.
static int cql_upload(prl_cql *s, int rounds, int64_t steps0, double alpha, float *out_loss, const CqlCall &dense, cudaStream_t st) {
    const prl_cql_cfg &c = s->cfg;
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
    CqlCall *hc = reinterpret_cast<CqlCall *>(tail + cql_call_offset(MR));
    *hc = dense;
    hc->slots = s->slots; hc->out_loss = out_loss;
    hc->decay = (float)(1.0 - c.lr * c.weight_decay);
    hc->alpha = (float)alpha;
    *reinterpret_cast<int *>(hc + 1) = 0;
    PRL_CUDA(cudaMemcpyAsync(s->scal, tail, s->tail_bytes, cudaMemcpyHostToDevice, st));
    PRL_CUDA(cudaEventRecord(s->tail_done[sb], st));
    return PRL_OK;
}

static int cql_run(prl_cql *s, prl_buf *buf, int rounds, int batch, cudaStream_t st) {
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
                cql_round(s, buf, batch, cs);
                e = cudaStreamEndCapture(cs, &graph);
            }
            if (e == cudaSuccess) e = cudaGraphInstantiate(&s->graph_exec[g], graph, 0);
            if (graph) cudaGraphDestroy(graph);
            cudaStreamDestroy(cs);
            if (e != cudaSuccess) { s->graph_exec[g] = nullptr; return fail(PRL_ECUDA, "prl_cql: graph capture failed: %s", cudaGetErrorString(e)); }
            s->graph_batch[g] = batch;
            if (buf) { s->graph_buf = buf->records; s->graph_dynamic = dynamic; }
        }
        for (int r = 0; r < rounds; r++) PRL_CUDA(cudaGraphLaunch(s->graph_exec[g], st));
    } else {
        for (int r = 0; r < rounds; r++) {
            int rc = cql_round(s, buf, batch, st);
            if (rc) return rc;
        }
    }
    PRL_CUDA(cudaGetLastError());
    s->adam_step += rounds;
    s->last_launches = (int64_t)s->launches_per_round * rounds;
    return PRL_OK;
}

extern "C" int prl_cql_learn(prl_cql *s, prl_buf *buf, int rounds, int batch, int64_t training_steps, double alpha, float *out_loss,
                             int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && out_loss, "null argument");
    const prl_cql_cfg &c = s->cfg;
    PRL_REQUIRE(rounds > 0 && rounds <= c.max_rounds && batch > 0 && batch <= c.max_batch, "rounds / batch outside the configured maxima");
    PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.obs_dim == c.obs_dim && buf->desc.n_actions == c.n_actions,
                "CQL needs a discrete-action buffer with obs_dim = %d and n_actions = %d", c.obs_dim, c.n_actions);
    PRL_REQUIRE(buf->shard_world <= 1, "the buffer is one shard of a multi-GPU buffer: CQL samples local buffers only");
    cudaStream_t st = (cudaStream_t)stream_;
    int rc = prl_buf_sample_indices(buf, rounds, batch, out_logical ? out_logical : s->logical, s->slots, stream_);
    if (rc) return rc;
    CqlCall dense;
    memset(&dense, 0, sizeof(dense));
    rc = cql_upload(s, rounds, training_steps + 1, alpha, out_loss, dense, st);   // PolicyLearner.learn counts the round first
    if (rc) return rc;
    return cql_run(s, buf, rounds, batch, st);
}

extern "C" int prl_cql_learn_batch(prl_cql *s, int batch, const float *state, const int32_t *action_id, const float *reward,
                                   const float *next_state, const uint8_t *terminated, const int32_t *curr_ids,
                                   const int32_t *next_ids, const int32_t *next_count, int64_t training_steps, double alpha,
                                   float *out_loss, void *stream_) {
    PRL_REQUIRE(s && state && action_id && reward && next_state && terminated && out_loss, "null argument");
    PRL_REQUIRE(batch > 0 && batch <= s->cfg.max_batch, "batch outside the configured maximum");
    cudaStream_t st = (cudaStream_t)stream_;
    CqlCall dense;
    memset(&dense, 0, sizeof(dense));
    dense.d_state = state; dense.d_next_state = next_state; dense.d_reward = reward; dense.d_action_id = action_id;
    dense.d_curr_ids = curr_ids; dense.d_next_ids = next_ids; dense.d_next_cnt = next_count; dense.d_term = terminated;
    int rc = cql_upload(s, 1, training_steps, alpha, out_loss, dense, st);
    if (rc) return rc;
    return cql_run(s, nullptr, 1, batch, st);
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

extern "C" int prl_cql_set_graph(prl_cql *s, int enable) {
    PRL_REQUIRE(s, "null handle");
    s->use_graph = enable != 0;
    return PRL_OK;
}
extern "C" int64_t prl_cql_last_launches(const prl_cql *s) { return s ? s->last_launches : -1; }
