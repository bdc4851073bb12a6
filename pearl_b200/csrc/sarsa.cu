// sarsa.cu — DeepSARSA (the on-policy member of DeepTDLearning), driven by PolicyLearner.learn over a replay buffer that
// stores the committed next action (PRL_BUF_NEXT_ACTION) or called directly on a caller's batch (PearlAgent.learn_batch),
// replacing
//   policy_learners/sequential_decision_making/deep_td_learning.py   forward, loss, learn_batch (target update FIRST,
//       MSE Bellman loss, AdamW step, reported mean |q - y|)
//   policy_learners/sequential_decision_making/deep_sarsa.py         get_next_state_values = Q_target(s', a')
//   neural_networks/sequential_decision_making/q_value_networks.py   VanillaQValueNetwork (state || one-hot action -> 1)
//
// One round: the soft target update in flagged rounds (with the CURRENT online parameters, before anything else), the
// online net over the B rows at the taken action, the target net over the B rows at (s', a') — B rows, no max over next
// actions, the available sets take no part — the Bellman target, the backward pass over B rows and AdamW(amsgrad).  The
// one-hot action is folded into layer 1 (k_fold).  Fixed launch sequence captured into a CUDA graph and replayed; unlike
// the other DQN-family handles, which keep one graph and re-capture when the batch changes, this one keeps a small cache
// of graphs keyed by (batch, buffer): an on-policy learner clears its buffer after every learn(), so its batch follows the
// episode length and repeats.  The AdamW step sizes, the decay factor and the per-round target-update flags are read
// through the per-call block, so prl_sarsa_set_lr needs no new capture.  fp32, fixed summation order, no float atomics:
// bit-reproducible run to run.
#include <math.h>

#include <new>

#include "common.cuh"
#include "dqn_family.cuh"
#include "gemm.cuh"

using namespace prl;

namespace {

constexpr int kMaxA = 255;   // next-action ids are stored as bytes
constexpr int kGraphs = 64;  // graphs kept per handle: an on-policy loop whose batch follows the episode length below
                             // batch_size (SARSA_method: 32) meets that many sizes; a graph of a round is a few KB

// per-call block the captured round reads through
struct SarsaCall {
    const int32_t *slots;                     // [rounds][B] (learn)
    float *out_loss;                          // [rounds]
    // learn_batch: the caller's dense batch
    const float *d_state, *d_next_state, *d_reward;
    const int32_t *d_action_id, *d_next_action_id;
    const uint8_t *d_term;
    float decay;                              // AdamW decoupled decay 1 - lr * weight_decay
};

// rows of one round: state, next state, reward, terminated, the taken action and the committed next action (bits 24..31
// of the record's flags word).  records == null: the caller's dense batch.
__global__ void k_sarsa_load(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, const SarsaCall *__restrict__ call,
                             const int *__restrict__ round_idx, int B, float *__restrict__ S, float *__restrict__ S2,
                             float *__restrict__ R, float *__restrict__ T, int *__restrict__ act, int *__restrict__ nact) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    if (!records) {
        for (int p = lane; p < obs; p += 32) {
            S[(size_t)w * obs + p] = call->d_state[(size_t)w * obs + p];
            S2[(size_t)w * obs + p] = call->d_next_state[(size_t)w * obs + p];
        }
        if (lane == 0) {
            act[w] = call->d_action_id[w];
            nact[w] = call->d_next_action_id[w];
            R[w] = call->d_reward[w];
            T[w] = call->d_term[w] ? 1.f : 0.f;
        }
        return;
    }
    const int32_t *slots = call->slots + (size_t)(*round_idx) * B;
    const uint32_t *r = records + (size_t)slots[w] * L.record_words;
    for (int p = lane; p < obs; p += 32) {
        S[(size_t)w * obs + p] = __uint_as_float(r[L.off_state + p]);
        S2[(size_t)w * obs + p] = __uint_as_float(r[L.off_next_state + p]);
    }
    if (lane == 0) {
        const uint32_t fl = r[L.off_flags];
        act[w] = (int)r[L.off_action];
        nact[w] = (int)(fl >> 24);
        R[w] = __uint_as_float(r[L.off_reward]);
        T[w] = (fl & 1u) ? 1.f : 0.f;
    }
}

// Bellman target and the MSE gradient, one thread per row, in the reference's operation order:
//   y = Q'(s', a') * gamma * (1 - terminated) + r;  dq = fl(2 / B) (q - y);  rowabs = |q - y|
__global__ void k_sarsa_target(int B, const float *__restrict__ q, const float *__restrict__ qt, const float *__restrict__ term,
                               const float *__restrict__ rew, float gamma, float *__restrict__ dq, float *__restrict__ rowabs) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float y = __fadd_rn(__fmul_rn(__fmul_rn(qt[b], gamma), __fsub_rn(1.f, term[b])), rew[b]);
    const float e = __fsub_rn(q[b], y);
    dq[b] = __fmul_rn(__fdiv_rn(2.f, (float)B), e);
    rowabs[b] = fabsf(e);
}

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_sarsa : DqnRounds<prl_sarsa, SarsaCall> {
    static constexpr const char *kFn = "prl_sarsa", *kName = "DeepSARSA";
    prl_sarsa_cfg cfg;
    int P;
    int W1, b1, W2, b2, W3, b3;
    float *q, *q_t, *q_m, *q_v, *q_x;
    // workspace
    float *S, *S2, *R, *T, *P1, *c1, *c2, *qa, *P1t, *c1t, *c2t, *qt, *dq, *rowabs, *dc2, *dc1, *grad;
    int *act, *nact;
    // graph cache, keyed by (dense batch, or the buffer's records and record stride, batch); the least recently used entry
    // makes room.  The stride is part of the key because a captured round bakes in the layout, and a new buffer may reuse
    // the storage address of an old one.
    struct Graph {
        cudaGraphExec_t exec = nullptr;
        const uint32_t *records = nullptr;
        int dense = 0, words = 0, batch = 0;
        int64_t used = 0;
    };
    Graph graphs[kGraphs];
    int64_t captures = 0, uses = 0;
    ~prl_sarsa() {
        for (Graph &g : graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
    }
    static int round(prl_sarsa *s, prl_buf *buf, int B, cudaStream_t st);
    int run(prl_buf *buf, int rounds, int batch, cudaStream_t st);   // hides DqnRounds::run: the cached-graph variant
};

static void sarsa_layout(prl_sarsa *s) {
    const prl_sarsa_cfg &c = s->cfg;
    const int D = c.obs_dim + c.n_actions;
    int o = 0;
    s->W1 = o; o += c.hidden1 * D; s->b1 = o; o += c.hidden1;
    s->W2 = o; o += c.hidden2 * c.hidden1; s->b2 = o; o += c.hidden2;
    s->W3 = o; o += c.hidden2; s->b3 = o; o += 1;
    s->P = o;
}

static int sarsa_check(const prl_sarsa_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->hidden1 > 0 && c->hidden2 > 0, "dimensions must be positive");
    PRL_REQUIRE(c->n_actions >= 1 && c->n_actions <= kMaxA, "n_actions must be in [1, %d]: next-action ids are stored as bytes", kMaxA);
    PRL_REQUIRE(c->target_update_freq > 0, "target_update_freq must be positive");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    const int64_t rows = c->max_batch > c->n_actions ? c->max_batch : c->n_actions;
    const int64_t elems = rows * (c->hidden1 > c->hidden2 ? c->hidden1 : c->hidden2);
    PRL_REQUIRE(elems < ((int64_t)1 << 31),
                "max(max_batch, n_actions) * max(hidden1, hidden2) = %lld must stay below 2^31 (32-bit element offsets)", (long long)elems);
    return PRL_OK;
}

extern "C" int64_t prl_sarsa_param_count(const prl_sarsa_cfg *c) {
    if (sarsa_check(c)) return -1;
    prl_sarsa t; t.cfg = *c; sarsa_layout(&t);
    return t.P;
}

// rows of the layer-1 / layer-2 activations: a round needs max_batch, q_values at least the A actions of one state
static int sarsa_qrows(const prl_sarsa_cfg &c) { return c.max_batch > c.n_actions ? c.max_batch : c.n_actions; }

// the workspace, in order; base == null: only its size
static int64_t sarsa_carve(prl_sarsa *s, void *base) {
    const prl_sarsa_cfg &c = s->cfg;
    const int64_t B = c.max_batch, O = c.obs_dim, H1 = c.hidden1, H2 = c.hidden2;
    Carve w{(char *)base};
    w(s->S, B * O); w(s->S2, B * O); w(s->R, B); w(s->T, B);
    const int64_t QR = sarsa_qrows(c);                                            // q_values reuses c1 / c2 for QR rows
    w(s->P1, B * H1); w(s->c1, QR * H1); w(s->c2, QR * H2); w(s->qa, B);        // online, at the taken action
    w(s->P1t, B * H1); w(s->c1t, B * H1); w(s->c2t, B * H2); w(s->qt, B);       // target, at the committed next action
    w(s->dq, B); w(s->rowabs, B); w(s->dc2, B * H2); w(s->dc1, B * H1); w(s->grad, s->P);
    w(s->act, B); w(s->nact, B);
    s->carve_tail(w, c.max_rounds, B);
    return w.bytes;
}
extern "C" int64_t prl_sarsa_workspace_bytes(const prl_sarsa_cfg *c) {
    if (sarsa_check(c)) return -1;
    prl_sarsa t; t.cfg = *c; sarsa_layout(&t);
    return sarsa_carve(&t, nullptr);
}

extern "C" int prl_sarsa_create(prl_sarsa **out, const prl_sarsa_cfg *cfg, float *w, float *w_target, float *exp_avg, float *exp_avg_sq,
                                float *max_exp_avg_sq, int64_t adam_step, void *workspace) {
    PRL_REQUIRE(out && w && w_target && exp_avg && exp_avg_sq && max_exp_avg_sq && workspace, "null argument");
    int rc = sarsa_check(cfg);
    if (rc) return rc;
    prl_sarsa *s = new (std::nothrow) prl_sarsa();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    sarsa_layout(s);
    s->q = w; s->q_t = w_target; s->q_m = exp_avg; s->q_v = exp_avg_sq; s->q_x = max_exp_avg_sq;
    s->adam_step = adam_step;
    sarsa_carve(s, workspace);
    return prl_sarsa::open(s, out);
}
extern "C" int prl_sarsa_destroy(prl_sarsa *s) { return prl_sarsa::destroy(s); }
extern "C" int64_t prl_sarsa_adam_step(const prl_sarsa *s) { return prl_sarsa::adam_step_of(s); }
extern "C" int prl_sarsa_set_adam_step(prl_sarsa *s, int64_t step) { return prl_sarsa::set_adam_step(s, step); }
extern "C" int prl_sarsa_set_lr(prl_sarsa *s, double lr) { return prl_sarsa::set_lr(s, lr); }
extern "C" int prl_sarsa_set_graph(prl_sarsa *s, int enable) { return prl_sarsa::set_graph(s, enable); }
extern "C" int64_t prl_sarsa_last_launches(const prl_sarsa *s) { return prl_sarsa::last_launches_of(s); }
extern "C" int64_t prl_sarsa_graph_captures(const prl_sarsa *s) { return s ? s->captures : -1; }

// the Q network at one action per row: layer 1 folded (state product + the action's W1 column), then two contractions
static void sarsa_fwd(const prl_sarsa *s, GemmLauncher &L, const float *net, const float *X, int m, const int *ids, float *P1, float *c1,
                      float *c2, float *out) {
    const prl_sarsa_cfg &c = s->cfg;
    const int O = c.obs_dim, D = O + c.n_actions, H1 = c.hidden1, H2 = c.hidden2, eb = 256;
    L.fwd(mat(X, O), m, net + s->W1, D, 0, net + s->b1, 0, H1, O, false, P1, H1, 0);
    k_fold<<<(unsigned)(((long long)m * H1 + eb - 1) / eb), eb, 0, L.st>>>(m, H1, P1, net + s->W1 + O, D, 0, ids, c1);
    L.fwd(mat(c1, H1), m, net + s->W2, H1, 0, net + s->b2, 0, H2, H1, true, c2, H2, 0);
    L.fwd(mat(c2, H2), m, net + s->W3, H2, 0, net + s->b3, 0, 1, H2, false, out, 1, 0);
}

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
int prl_sarsa::round(prl_sarsa *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_sarsa_cfg &c = s->cfg;
    const int O = c.obs_dim, A = c.n_actions, D = O + A, H1 = c.hidden1, H2 = c.hidden2;
    // the decay factor is overridden by call->decay (k_adamw's decay pointer)
    const AdamHp h = adam_hp(0.0, c.beta1, c.beta2, c.eps, c.weight_decay);
    GemmLauncher L; L.st = st;
    const float *w = s->q;
    float *g = s->grad;
    const int eb = 256;
    int small = 0;
    k_sarsa_load<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf ? buf->records : nullptr, buf ? buf->lay : prl_buf_layout{}, O, s->call,
                                                       s->round_idx, B, s->S, s->S2, s->R, s->T, s->act, s->nact);
    // ---------------- target update first, with the current online parameters (flagged rounds only)
    k_soft_update_flagged<<<(s->P + eb - 1) / eb, eb, 0, st>>>(s->P, s->q, s->q_t, (float)c.tau, (float)(1.0 - c.tau), s->target_on,
                                                               s->round_idx);
    small += 2;
    // ---------------- online net at the taken action (kept for the backward pass); target net at (s', a')
    sarsa_fwd(s, L, w, s->S, B, s->act, s->P1, s->c1, s->c2, s->qa);
    sarsa_fwd(s, L, s->q_t, s->S2, B, s->nact, s->P1t, s->c1t, s->c2t, s->qt);
    small += 2;
    // ---------------- Bellman target and the MSE gradient
    k_sarsa_target<<<(B + 127) / 128, 128, 0, st>>>(B, s->qa, s->qt, s->T, s->R, (float)c.gamma, s->dq, s->rowabs);
    small++;
    // ---------------- backward through the online net over B rows
    L.bwd_w(s->dq, 1, 0, B, 1, mat(s->c2, H2), H2, g + s->W3, H2, 0, g + s->b3, 0);
    k_head_bwd<<<(unsigned)(((long long)B * H2 + eb - 1) / eb), eb, 0, st>>>(B, H2, s->dq, w + s->W3, 0, s->c2, s->dc2);
    L.bwd_w(s->dc2, H2, 0, B, H2, mat(s->c1, H1), H1, g + s->W2, H1, 0, g + s->b2, 0);
    L.bwd_x(s->dc2, H2, 0, B, H2, w + s->W2, H1, 0, 0, H1, s->dc1, H1, 0, s->c1, H1, 0, false);
    L.bwd_w(s->dc1, H1, 0, B, H1, mat(s->S, O), O, g + s->W1, D, 0, g + s->b1, 0);                   // state columns + b1
    k_fold_w1a_grad<<<(H1 * A + eb - 1) / eb, eb, 0, st>>>(B, A, H1, s->act, s->dc1, g + s->W1 + O, D, 0);
    small += 2;
    // ---------------- AdamW(amsgrad); the target was updated at the start of the round
    k_adamw<<<(s->P + eb - 1) / eb, eb, 0, st>>>(s->P, s->q, s->q_m, s->q_v, s->q_x, g, h, s->scal, s->round_idx, nullptr, 0.f, 0.f,
                                                &s->call->decay);
    k_round_report<<<1, 256, 0, st>>>(B, s->rowabs, s->call, s->round_idx);
    small += 2;
    s->launches_per_round = L.count + small;
    return PRL_OK;
}

// `rounds` rounds: replays of the cached graph of this (batch, buffer), captured on a miss, or eager launches
int prl_sarsa::run(prl_buf *buf, int rounds, int batch, cudaStream_t st) {
    if (use_graph) {
        const int dense = buf ? 0 : 1;
        const uint32_t *rec = buf ? buf->records : nullptr;
        const int words = buf ? buf->lay.record_words : 0;
        Graph *hit = nullptr;
        for (Graph &e : graphs)
            if (e.exec && e.dense == dense && e.batch == batch && e.records == rec && e.words == words) { hit = &e; break; }
        if (!hit) {
            for (Graph &e : graphs) if (!e.exec) { hit = &e; break; }
            if (!hit) {
                hit = &graphs[0];
                for (Graph &e : graphs) if (e.used < hit->used) hit = &e;
            }
            // capture_graph releases the evicted graph (freed once its launches in flight complete)
            int rc = capture_graph(&hit->exec, kFn, [&](cudaStream_t cs) { return round(this, buf, batch, cs); });
            if (rc) return rc;
            hit->dense = dense; hit->records = rec; hit->words = words; hit->batch = batch;
            captures++;
        }
        hit->used = ++uses;
        for (int r = 0; r < rounds; r++) PRL_CUDA(cudaGraphLaunch(hit->exec, st));
    } else {
        for (int r = 0; r < rounds; r++) {
            int rc = round(this, buf, batch, st);
            if (rc) return rc;
        }
    }
    PRL_CUDA(cudaGetLastError());
    adam_step += rounds;
    last_launches = (int64_t)launches_per_round * rounds;
    return PRL_OK;
}

extern "C" int prl_sarsa_learn(prl_sarsa *s, prl_buf *buf, int rounds, int batch, int64_t training_steps, float *out_loss,
                               int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf, "null argument");
    PRL_REQUIRE(buf->desc.flags & PRL_BUF_NEXT_ACTION,
                "DeepSARSA needs the committed next action of every transition: learn over a B200SARSAReplayBuffer "
                "(a buffer created with PRL_BUF_NEXT_ACTION)");
    return prl_sarsa::learn(s, buf, rounds, batch, training_steps, out_loss, out_logical, SarsaCall{}, stream_);
}

extern "C" int prl_sarsa_learn_batch(prl_sarsa *s, int batch, const float *state, const int32_t *action_id, const float *reward,
                                     const float *next_state, const int32_t *next_action_id, const uint8_t *terminated,
                                     int64_t training_steps, float *out_loss, void *stream_) {
    PRL_REQUIRE(s && state && action_id && reward && next_state && next_action_id && terminated && out_loss, "null argument");
    SarsaCall dense{};
    dense.d_state = state; dense.d_next_state = next_state; dense.d_reward = reward; dense.d_action_id = action_id;
    dense.d_next_action_id = next_action_id; dense.d_term = terminated;
    return prl_sarsa::learn_batch(s, batch, training_steps, out_loss, dense, stream_);
}

// Q(s, a) for every action: the online forward of the round on n rows (chunks of max_batch rows through the workspace)
extern "C" int prl_sarsa_q_values(prl_sarsa *s, int n, const float *state, int target, float *out_q, void *stream_) {
    PRL_REQUIRE(s && state && out_q, "null argument");
    if (n <= 0) return PRL_OK;
    const prl_sarsa_cfg &c = s->cfg;
    const int O = c.obs_dim, A = c.n_actions, D = O + A, H1 = c.hidden1, H2 = c.hidden2, eb = 256;
    const float *w = target ? s->q_t : s->q;
    GemmLauncher L; L.st = (cudaStream_t)stream_;
    // c1 / c2 hold max(max_batch, A) (state, action) rows: chunks of that many rows over A, at least one state row
    const int rows = sarsa_qrows(c) / A;
    for (int r0 = 0; r0 < n; r0 += rows) {
        const int m = n - r0 < rows ? n - r0 : rows, mA = m * A;
        L.fwd(mat(state + (size_t)r0 * O, O), m, w + s->W1, D, 0, w + s->b1, 0, H1, O, false, s->P1, H1, 0);
        k_fold_expand<<<(unsigned)(((long long)mA * H1 + eb - 1) / eb), eb, 0, L.st>>>(m, A, H1, s->P1, w + s->W1 + O, D, 0, nullptr, s->c1);
        L.fwd(mat(s->c1, H1), mA, w + s->W2, H1, 0, w + s->b2, 0, H2, H1, true, s->c2, H2, 0);
        L.fwd(mat(s->c2, H2), mA, w + s->W3, H2, 0, w + s->b3, 0, 1, H2, false, out_q + (size_t)r0 * A, 1, 0);
    }
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}
