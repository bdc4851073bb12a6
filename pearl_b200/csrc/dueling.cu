// dueling.cu — dueling DQN / DoubleDQN (DeepQLearning / DoubleDQN built with network_type=DuelingQValueNetwork), driven
// by PolicyLearner.learn or called directly on a caller's batch (PearlAgent.learn_batch), replacing
//   neural_networks/sequential_decision_making/q_value_networks.py   DuelingQValueNetwork.get_q_values
//   policy_learners/sequential_decision_making/deep_td_learning.py   forward, loss, learn_batch (target update FIRST,
//       MSE Bellman loss, AdamW step, reported mean |q - y|)
//   policy_learners/sequential_decision_making/deep_q_learning.py    get_next_state_values (max over available slots)
//   policy_learners/sequential_decision_making/double_dqn.py         get_next_state_values (online first argmax, target value)
//
// The network is three MLPs (Linear+ReLU, Linear+ReLU, Linear): the trunk state_arch (obs -> F, no ReLU on the feature),
// value_arch (F -> 1) and advantage_arch (F || one-hot action -> 1).  get_q_values returns fl(fl(V + Adv(a)) - mean Adv)
// where the mean runs over a set that depends on the caller:
//   online q (forward):   the A current slots c_b[k], padding (id 0) included, the unavailable mask ignored; or, when a
//                         dense batch has no current sets, the query action alone: q = fl(fl(V + Adv) - Adv)
//   DQN target:           all A next slots (masked ones with the id they hold, 0 as the reference pads), then masked max
//   DoubleDQN target:     the online net over all A next slots picks a* (first argmax over the available ones); the target
//                         net is then called with the single query a*, so V' = fl(fl(V_t + Adv_t(a*)) - Adv_t(a*))
//   q_values (act):       the caller's id set, e.g. the available actions only
// So dq reaches the advantage net as +dq on the taken-action row and -dq / A on every current slot (zero in query-alone
// mode), and the value net as dq.
//
// One round: the soft target update in flagged rounds (with the CURRENT online parameters, before anything else), the
// online net on the B states with the advantage over B*(A+1) rows (slots 0..A-1 = current set, slot A = taken action), the
// target net (and, for DoubleDQN, the online net) on the B next states with the advantage over the B*A next slots, the
// Bellman target and slot gradients, the backward pass (advantage rows summed per row, then through the trunk with the
// value head's part added) and AdamW(amsgrad).  Fixed launch sequence, captured once per (batch, buffer) into a CUDA graph
// and replayed (DESIGN.md §3.4).  The AdamW step sizes, the decay factor, the per-round target-update flags and the
// query-alone switch are read through the per-call block, so prl_duel_set_lr needs no new capture.  fp32, fixed summation
// order, no float atomics: bit-reproducible run to run.
#include <limits.h>
#include <math.h>

#include <new>

#include "common.cuh"
#include "gemm.cuh"

using namespace prl;

namespace {

constexpr int kMaxA = 255;   // next-action ids are stored as bytes

// per-call block the captured round reads through
struct DuelCall {
    const int32_t *slots;                     // [rounds][B] (learn)
    float *out_loss;                          // [rounds]
    // learn_batch: the caller's dense batch
    const float *d_state, *d_next_state, *d_reward;
    const int32_t *d_action_id;
    const int32_t *d_curr_ids;                // [B][A] current slot ids
    const int32_t *d_next_ids;                // [B][A] next slot ids; null: slot k holds k
    const uint8_t *d_next_unavail;            // [B][A] 1 = unavailable; null: every slot available
    const uint8_t *d_term;
    float decay;                              // AdamW decoupled decay 1 - lr * weight_decay
    int query_alone;                          // the online mean runs over the query action alone (no current sets)
};

// mean over K slot values, one warp per row: per-lane sums in slot order, a fixed xor tree, then / K (torch.mean)
__device__ __forceinline__ float slot_mean(const float *a, int K, int lane) {
    float s = 0.f;
    for (int k = lane; k < K; k += 32) s += a[k];
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return __fdiv_rn(s, (float)K);
}

__device__ __forceinline__ float duel_q(float V, float adv, float mean) { return __fsub_rn(__fadd_rn(V, adv), mean); }

// rows of one round: state, next state, reward, terminated, the id and unavailable flag of every next slot (slots at or
// beyond the stored count read as id 0, as the reference pads), and the A + 1 online slots: cids[b][k] = c_b[k] for k < A,
// cids[b][A] = the taken action.  records == null: pack the caller's dense batch.  The ring stores no current action sets:
// every action, as B200ReplayBuffer.sample reports.
__global__ void k_duel_load(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int A, int dynamic,
                            const DuelCall *__restrict__ call, const int *__restrict__ round_idx, int B, float *__restrict__ S,
                            float *__restrict__ S2, float *__restrict__ R, float *__restrict__ T, int *__restrict__ ids,
                            int *__restrict__ un, int *__restrict__ cids) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    int *crow = cids + (size_t)w * (A + 1);
    int *irow = ids + (size_t)w * A, *urow = un + (size_t)w * A;
    if (!records) {
        for (int p = lane; p < obs; p += 32) {
            S[(size_t)w * obs + p] = call->d_state[(size_t)w * obs + p];
            S2[(size_t)w * obs + p] = call->d_next_state[(size_t)w * obs + p];
        }
        const int32_t *nid = call->d_next_ids, *cid = call->d_curr_ids;
        const uint8_t *nu = call->d_next_unavail;
        for (int k = lane; k < A; k += 32) {
            irow[k] = nid ? nid[(size_t)w * A + k] : k;
            urow[k] = nu ? (nu[(size_t)w * A + k] ? 1 : 0) : 0;
            crow[k] = cid ? cid[(size_t)w * A + k] : k;
        }
        if (lane == 0) {
            crow[A] = call->d_action_id[w];
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
    const uint32_t fl = r[L.off_flags];
    const int cnt = dynamic ? min((int)((fl >> 8) & 0xffffu), A) : A;
    const uint8_t *id8 = reinterpret_cast<const uint8_t *>(r + L.off_avail);
    for (int k = lane; k < A; k += 32) {
        irow[k] = dynamic ? (k < cnt ? (int)id8[k] : 0) : k;
        urow[k] = k < cnt ? 0 : 1;
        crow[k] = k;
    }
    if (lane == 0) {
        crow[A] = (int)r[L.off_action];
        R[w] = __uint_as_float(r[L.off_reward]);
        T[w] = (fl & 1u) ? 1.f : 0.f;
    }
}

// Bellman target and the loss gradients.  One warp per row b; lane l handles slots l, l + 32, ...
//   next Q(s', k) = fl(fl(V'(s') + Adv'(s', k)) - mean over the A next slots of Adv'(s', .))
//   DQN:        V = max over available next slots of Q_target(s', .)
//   DoubleDQN:  a* = first argmax over available next slots of Q_online(s', .), V = fl(fl(V_t + Adv_t(a*)) - Adv_t(a*))
//   y = V * gamma * (1 - terminated) + r;  q = fl(fl(V(s) + Adv(s, a)) - mean over the current slots (or Adv(s, a)));
//   dq = fl(2 / B) (q - y) (MSELoss): dV = dq, dAdv[b][A] = dq, dAdv[b][k < A] = -dq / A  (both 0 in query-alone mode)
// vo / ao: online V [B] and advantages [B][A + 1]; vt / at (vn / an): target (online) next V [B] and advantages [B][A].
__global__ void __launch_bounds__(128) k_duel_target(int B, int A, int dbl, const float *__restrict__ vo, const float *__restrict__ ao,
                                                     const float *__restrict__ vt, const float *__restrict__ at,
                                                     const float *__restrict__ vn, const float *__restrict__ an,
                                                     const int *__restrict__ un, const float *__restrict__ term,
                                                     const float *__restrict__ rew, const DuelCall *__restrict__ call, float gamma,
                                                     float *__restrict__ dv, float *__restrict__ dadv, float *__restrict__ rowabs) {
    const int lane = threadIdx.x & 31, b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= B) return;
    const int *u = un + (size_t)b * A;
    const float *sa = (dbl ? an : at) + (size_t)b * A;
    const float sv = dbl ? vn[b] : vt[b];
    const float sm = slot_mean(sa, A, lane);
    float best = -INFINITY;
    int bk = INT_MAX;
    for (int k = lane; k < A; k += 32) {
        const float v = u[k] ? -INFINITY : duel_q(sv, sa[k], sm);
        if (v > best || (v == best && k < bk)) { best = v; bk = k; }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int ok = __shfl_xor_sync(0xffffffffu, bk, o);
        if (ov > best || (ov == best && ok < bk)) { best = ov; bk = ok; }
    }
    float V = best;
    if (dbl) {
        const float a = at[(size_t)b * A + (bk == INT_MAX ? 0 : bk)];
        V = duel_q(vt[b], a, a);
    }
    const float *ar = ao + (size_t)b * (A + 1);
    const int qa = call->query_alone;
    const float cm = qa ? ar[A] : slot_mean(ar, A, lane);
    const float q = duel_q(vo[b], ar[A], cm);
    const float y = __fadd_rn(__fmul_rn(__fmul_rn(V, gamma), __fsub_rn(1.f, term[b])), rew[b]);
    const float e = __fsub_rn(q, y);
    const float dq = __fmul_rn(__fdiv_rn(2.f, (float)B), e);
    float *d = dadv + (size_t)b * (A + 1);
    const float ds = qa ? 0.f : __fdiv_rn(-dq, (float)A);
    for (int k = lane; k < A; k += 32) d[k] = ds;
    if (lane == 0) {
        d[A] = qa ? 0.f : dq;
        dv[b] = dq;
        rowabs[b] = fabsf(e);
    }
}

// Q values over a caller's id set: out[b][k] = fl(fl(V[b] + adv[b][k]) - mean_k adv[b][.]), one warp per row
__global__ void __launch_bounds__(128) k_duel_q(int n, int K, const float *__restrict__ V, const float *__restrict__ adv,
                                                float *__restrict__ out) {
    const int lane = threadIdx.x & 31, b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= n) return;
    const float *a = adv + (size_t)b * K;
    const float m = slot_mean(a, K, lane);
    for (int k = lane; k < K; k += 32) out[(size_t)b * K + k] = duel_q(V[b], a[k], m);
}

}  // namespace

// ------------------------------------------------------------------ host side
// one MLP of the network in the flat vector: W1[h1][in] b1 W2[h2][h1] b2 W3[out][h2] b3
struct DuelMlp { int W1, b1, W2, b2, W3, b3, in, h1, h2, out; };
// activations of one forward pass on m rows with K advantage slots per row
struct DuelAct { float *t1, *t2, *f, *v1, *v2, *V, *Pa, *a1, *a2, *adv; };

struct prl_duel {
    prl_duel_cfg cfg;
    int P;
    DuelMlp st, va, ad;
    float *q, *q_t, *q_m, *q_v, *q_x;
    int64_t adam_step;
    // workspace
    float *S, *S2, *R, *T;
    DuelAct on, nx;                           // online pass (kept for the backward pass); next-state pass scratch
    float *Vt, *At, *Vn, *An;                 // next-state V / advantages of the target and (DoubleDQN) online net
    float *dV, *dAdv, *rowabs, *da2, *da1, *dPa, *dv2, *dv1, *df, *dt2, *dt1, *grad;
    int *ids, *un, *cids;
    int32_t *slots, *logical;
    float2 *scal;
    int *target_on;
    DuelCall *call;
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
static size_t duel_call_offset(int MR) { return ((size_t)MR * 12 + 7) / 8 * 8; }
static size_t duel_tail_bytes(int MR) { return duel_call_offset(MR) + sizeof(DuelCall) + 4; }

static void mlp_at(DuelMlp &m, int &o, int in, int h1, int h2, int out) {
    m.in = in; m.h1 = h1; m.h2 = h2; m.out = out;
    m.W1 = o; o += h1 * in; m.b1 = o; o += h1;
    m.W2 = o; o += h2 * h1; m.b2 = o; o += h2;
    m.W3 = o; o += out * h2; m.b3 = o; o += out;
}

static void duel_layout(prl_duel *s) {
    const prl_duel_cfg &c = s->cfg;
    int o = 0;
    mlp_at(s->st, o, c.obs_dim, c.state_h1, c.state_h2, c.feature_dim);
    mlp_at(s->va, o, c.feature_dim, c.value_h1, c.value_h2, 1);
    mlp_at(s->ad, o, c.feature_dim + c.n_actions, c.adv_h1, c.adv_h2, 1);
    s->P = o;
}

static int duel_check(const prl_duel_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->feature_dim > 0 && c->state_h1 > 0 && c->state_h2 > 0 && c->value_h1 > 0 && c->value_h2 > 0 &&
                c->adv_h1 > 0 && c->adv_h2 > 0, "dimensions must be positive");
    PRL_REQUIRE(c->n_actions >= 1 && c->n_actions <= kMaxA, "n_actions must be in [1, %d]: next-action ids are stored as bytes", kMaxA);
    PRL_REQUIRE(c->target_update_freq > 0, "target_update_freq must be positive");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    return PRL_OK;
}

extern "C" int64_t prl_duel_param_count(const prl_duel_cfg *c) {
    if (duel_check(c)) return -1;
    prl_duel t; t.cfg = *c; duel_layout(&t);
    return t.P;
}

struct DuelWs { int64_t off[48]; int64_t total; };
static DuelWs duel_ws(const prl_duel_cfg *c, int P) {
    DuelWs w; int64_t o = 0; int k = 0;
    const int64_t B = c->max_batch, O = c->obs_dim, A = c->n_actions, F = c->feature_dim, BA = B * A, BA1 = B * (A + 1);
    auto add = [&](int64_t words) { w.off[k++] = o; o = al64(o + words * 4); };
    add(B * O); add(B * O); add(B); add(B);                                               // S S2 R T
    for (int64_t rows : {BA1, BA}) {                                                      // online pass, next-state pass
        add(B * c->state_h1); add(B * c->state_h2); add(B * F);                           // t1 t2 f
        add(B * c->value_h1); add(B * c->value_h2); add(B);                               // v1 v2 V
        add(B * c->adv_h1); add(rows * c->adv_h1); add(rows * c->adv_h2); add(rows);      // Pa a1 a2 adv
    }
    add(B); add(BA); add(B); add(BA);                                                     // Vt At Vn An
    add(B); add(BA1); add(B);                                                             // dV dAdv rowabs
    add(BA1 * c->adv_h2); add(BA1 * c->adv_h1); add(B * c->adv_h1);                       // da2 da1 dPa
    add(B * c->value_h2); add(B * c->value_h1); add(B * F);                               // dv2 dv1 df
    add(B * c->state_h2); add(B * c->state_h1); add(P);                                   // dt2 dt1 grad
    add(BA); add(BA); add(BA1);                                                           // ids un cids (int32)
    add((int64_t)c->max_rounds * B); add((int64_t)c->max_rounds * B);                    // slots logical (int32)
    add(((int64_t)duel_tail_bytes(c->max_rounds) + 3) / 4);                               // scal | target_on | call | round_idx
    w.total = o;
    return w;
}
extern "C" int64_t prl_duel_workspace_bytes(const prl_duel_cfg *c) {
    if (duel_check(c)) return -1;
    prl_duel t; t.cfg = *c; duel_layout(&t);
    return duel_ws(c, t.P).total;
}

extern "C" int prl_duel_create(prl_duel **out, const prl_duel_cfg *cfg, float *w, float *w_target, float *exp_avg, float *exp_avg_sq,
                               float *max_exp_avg_sq, int64_t adam_step, void *workspace) {
    PRL_REQUIRE(out && w && w_target && exp_avg && exp_avg_sq && max_exp_avg_sq && workspace, "null argument");
    int rc = duel_check(cfg);
    if (rc) return rc;
    prl_duel *s = new (std::nothrow) prl_duel();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    duel_layout(s);
    s->q = w; s->q_t = w_target; s->q_m = exp_avg; s->q_v = exp_avg_sq; s->q_x = max_exp_avg_sq;
    s->adam_step = adam_step;
    DuelWs ws = duel_ws(cfg, s->P);
    char *b = (char *)workspace;
    float **f[] = {&s->S, &s->S2, &s->R, &s->T,
                   &s->on.t1, &s->on.t2, &s->on.f, &s->on.v1, &s->on.v2, &s->on.V, &s->on.Pa, &s->on.a1, &s->on.a2, &s->on.adv,
                   &s->nx.t1, &s->nx.t2, &s->nx.f, &s->nx.v1, &s->nx.v2, &s->nx.V, &s->nx.Pa, &s->nx.a1, &s->nx.a2, &s->nx.adv,
                   &s->Vt, &s->At, &s->Vn, &s->An, &s->dV, &s->dAdv, &s->rowabs, &s->da2, &s->da1, &s->dPa, &s->dv2, &s->dv1,
                   &s->df, &s->dt2, &s->dt1, &s->grad};
    int k = 0;
    for (auto p : f) *p = (float *)(b + ws.off[k++]);
    s->ids = (int *)(b + ws.off[k++]); s->un = (int *)(b + ws.off[k++]); s->cids = (int *)(b + ws.off[k++]);
    s->slots = (int32_t *)(b + ws.off[k++]); s->logical = (int32_t *)(b + ws.off[k++]);
    char *tail = b + ws.off[k++];
    const int MR = cfg->max_rounds;
    s->scal = (float2 *)tail;
    s->target_on = (int *)(tail + (size_t)MR * 8);
    s->call = (DuelCall *)(tail + duel_call_offset(MR));
    s->round_idx = (int *)(s->call + 1);
    s->tail_bytes = duel_tail_bytes(MR);
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
        return fail(PRL_ECUDA, "prl_duel_create: %s", cudaGetErrorString(e));
    }
    *out = s;
    return PRL_OK;
}
extern "C" int prl_duel_destroy(prl_duel *s) {
    if (!s) return PRL_OK;
    for (int i = 0; i < 2; i++) { cudaEventSynchronize(s->tail_done[i]); cudaEventDestroy(s->tail_done[i]); cudaFreeHost(s->tail_host[i]); }
    for (int i = 0; i < 2; i++) if (s->graph_exec[i]) cudaGraphExecDestroy(s->graph_exec[i]);
    delete s;
    return PRL_OK;
}
extern "C" int64_t prl_duel_adam_step(const prl_duel *s) { return s ? s->adam_step : -1; }
extern "C" int prl_duel_set_adam_step(prl_duel *s, int64_t step) {
    PRL_REQUIRE(s, "null handle");
    PRL_REQUIRE(step >= 0, "the AdamW step count must be non-negative");
    s->adam_step = step;
    return PRL_OK;
}

extern "C" int prl_duel_set_lr(prl_duel *s, double lr) {
    PRL_REQUIRE(s, "null handle");
    PRL_REQUIRE(lr >= 0.0, "the learning rate must be non-negative");
    s->cfg.lr = lr;
    return PRL_OK;
}

// the network `net` on m states X: trunk feature, V, and the advantage at K slots per row (ids [m][K]; null: slot k holds
// k).  The feature part of advantage layer 1 is computed once per row and expanded per slot.  Returns the small launches.
static int duel_fwd(const prl_duel *s, GemmLauncher &L, const float *net, const float *X, int m, int K, const int *ids, const DuelAct &a) {
    const DuelMlp &st = s->st, &va = s->va, &ad = s->ad;
    const int O = st.in, F = st.out, mK = m * K, eb = 256;
    L.fwd(mat(X, O), m, net + st.W1, O, 0, net + st.b1, 0, st.h1, O, true, a.t1, st.h1, 0);
    L.fwd(mat(a.t1, st.h1), m, net + st.W2, st.h1, 0, net + st.b2, 0, st.h2, st.h1, true, a.t2, st.h2, 0);
    L.fwd(mat(a.t2, st.h2), m, net + st.W3, st.h2, 0, net + st.b3, 0, F, st.h2, false, a.f, F, 0);
    L.fwd(mat(a.f, F), m, net + va.W1, F, 0, net + va.b1, 0, va.h1, F, true, a.v1, va.h1, 0);
    L.fwd(mat(a.v1, va.h1), m, net + va.W2, va.h1, 0, net + va.b2, 0, va.h2, va.h1, true, a.v2, va.h2, 0);
    L.fwd(mat(a.v2, va.h2), m, net + va.W3, va.h2, 0, net + va.b3, 0, 1, va.h2, false, a.V, 1, 0);
    L.fwd(mat(a.f, F), m, net + ad.W1, ad.in, 0, net + ad.b1, 0, ad.h1, F, false, a.Pa, ad.h1, 0);
    k_fold_expand<<<(unsigned)(((long long)mK * ad.h1 + eb - 1) / eb), eb, 0, L.st>>>(m, K, ad.h1, a.Pa, net + ad.W1 + F, ad.in, 0, ids, a.a1);
    L.fwd(mat(a.a1, ad.h1), mK, net + ad.W2, ad.h1, 0, net + ad.b2, 0, ad.h2, ad.h1, true, a.a2, ad.h2, 0);
    L.fwd(mat(a.a2, ad.h2), mK, net + ad.W3, ad.h2, 0, net + ad.b3, 0, 1, ad.h2, false, a.adv, 1, 0);
    return 1;
}

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
static int duel_round(prl_duel *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_duel_cfg &c = s->cfg;
    const DuelMlp &sa = s->st, &va = s->va, &ad = s->ad;
    const int O = c.obs_dim, A = c.n_actions, F = c.feature_dim, BA1 = B * (A + 1);
    // the decay factor is overridden by call->decay (k_adamw's decay pointer)
    const AdamHp h = adam_hp(0.0, c.beta1, c.beta2, c.eps, c.weight_decay);
    GemmLauncher L; L.st = st;
    const float *w = s->q;
    float *g = s->grad;
    const DuelAct &on = s->on;
    const int eb = 256;
    int small = 0;
    const int dynamic = (buf && (buf->desc.flags & PRL_BUF_DYNAMIC_ACTIONS)) ? 1 : 0;
    k_duel_load<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf ? buf->records : nullptr, buf ? buf->lay : prl_buf_layout{}, O, A, dynamic,
                                                      s->call, s->round_idx, B, s->S, s->S2, s->R, s->T, s->ids, s->un, s->cids);
    // ---------------- target update first, with the current online parameters (flagged rounds only)
    k_soft_update_flagged<<<(s->P + eb - 1) / eb, eb, 0, st>>>(s->P, s->q, s->q_t, (float)c.tau, (float)(1.0 - c.tau), s->target_on,
                                                               s->round_idx);
    small += 2;
    // ---------------- online net: the A current slots and the taken action (kept for the backward pass)
    small += duel_fwd(s, L, w, s->S, B, A + 1, s->cids, on);
    // ---------------- DoubleDQN: the online net over the next slots (greedy slot); then the target net over them
    DuelAct nx = s->nx;
    if (c.double_dqn) {
        nx.V = s->Vn; nx.adv = s->An;
        small += duel_fwd(s, L, w, s->S2, B, A, s->ids, nx);
    }
    nx.V = s->Vt; nx.adv = s->At;
    small += duel_fwd(s, L, s->q_t, s->S2, B, A, s->ids, nx);
    // ---------------- Bellman target and the gradients at V and at the advantage slots
    k_duel_target<<<(B * 32 + 127) / 128, 128, 0, st>>>(B, A, c.double_dqn, on.V, on.adv, s->Vt, s->At, s->Vn, s->An, s->un, s->T, s->R,
                                                       s->call, (float)c.gamma, s->dV, s->dAdv, s->rowabs);
    small++;
    // ---------------- advantage net backward over B*(A+1) rows; the slots' layer-1 gradients summed per row
    L.bwd_w(s->dAdv, 1, 0, BA1, 1, mat(on.a2, ad.h2), ad.h2, g + ad.W3, ad.h2, 0, g + ad.b3, 0);
    k_head_bwd<<<(BA1 * ad.h2 + eb - 1) / eb, eb, 0, st>>>(BA1, ad.h2, s->dAdv, w + ad.W3, 0, on.a2, s->da2);
    L.bwd_w(s->da2, ad.h2, 0, BA1, ad.h2, mat(on.a1, ad.h1), ad.h1, g + ad.W2, ad.h1, 0, g + ad.b2, 0);
    L.bwd_x(s->da2, ad.h2, 0, BA1, ad.h2, w + ad.W2, ad.h1, 0, 0, ad.h1, s->da1, ad.h1, 0, on.a1, ad.h1, 0, false);
    k_slot_rowsum<<<(B * ad.h1 + eb - 1) / eb, eb, 0, st>>>(B, A + 1, ad.h1, s->da1, s->dPa);
    L.bwd_w(s->dPa, ad.h1, 0, B, ad.h1, mat(on.f, F), F, g + ad.W1, ad.in, 0, g + ad.b1, 0);             // feature columns + b1
    k_fold_w1a_grad<<<(ad.h1 * A + eb - 1) / eb, eb, 0, st>>>(BA1, A, ad.h1, s->cids, s->da1, g + ad.W1 + F, ad.in, 0);
    L.bwd_x(s->dPa, ad.h1, 0, B, ad.h1, w + ad.W1, ad.in, 0, 0, F, s->df, F, 0, nullptr, 0, 0, false);    // df = dPa W1a[:, :F]
    small += 3;
    // ---------------- value net backward over B rows; its feature gradient is added to df
    L.bwd_w(s->dV, 1, 0, B, 1, mat(on.v2, va.h2), va.h2, g + va.W3, va.h2, 0, g + va.b3, 0);
    k_head_bwd<<<(B * va.h2 + eb - 1) / eb, eb, 0, st>>>(B, va.h2, s->dV, w + va.W3, 0, on.v2, s->dv2);
    L.bwd_w(s->dv2, va.h2, 0, B, va.h2, mat(on.v1, va.h1), va.h1, g + va.W2, va.h1, 0, g + va.b2, 0);
    L.bwd_x(s->dv2, va.h2, 0, B, va.h2, w + va.W2, va.h1, 0, 0, va.h1, s->dv1, va.h1, 0, on.v1, va.h1, 0, false);
    L.bwd_w(s->dv1, va.h1, 0, B, va.h1, mat(on.f, F), F, g + va.W1, F, 0, g + va.b1, 0);
    L.bwd_x(s->dv1, va.h1, 0, B, va.h1, w + va.W1, F, 0, 0, F, s->df, F, 0, nullptr, 0, 0, true);
    small++;
    // ---------------- trunk backward (the feature is a Linear output: no ReLU mask on df)
    L.bwd_w(s->df, F, 0, B, F, mat(on.t2, sa.h2), sa.h2, g + sa.W3, sa.h2, 0, g + sa.b3, 0);
    L.bwd_x(s->df, F, 0, B, F, w + sa.W3, sa.h2, 0, 0, sa.h2, s->dt2, sa.h2, 0, on.t2, sa.h2, 0, false);
    L.bwd_w(s->dt2, sa.h2, 0, B, sa.h2, mat(on.t1, sa.h1), sa.h1, g + sa.W2, sa.h1, 0, g + sa.b2, 0);
    L.bwd_x(s->dt2, sa.h2, 0, B, sa.h2, w + sa.W2, sa.h1, 0, 0, sa.h1, s->dt1, sa.h1, 0, on.t1, sa.h1, 0, false);
    L.bwd_w(s->dt1, sa.h1, 0, B, sa.h1, mat(s->S, O), O, g + sa.W1, O, 0, g + sa.b1, 0);
    // ---------------- AdamW(amsgrad); the target was updated at the start of the round
    k_adamw<<<(s->P + eb - 1) / eb, eb, 0, st>>>(s->P, s->q, s->q_m, s->q_v, s->q_x, g, h, s->scal, s->round_idx, nullptr, 0.f, 0.f,
                                                &s->call->decay);
    k_round_report<<<1, 256, 0, st>>>(B, s->rowabs, s->call, s->round_idx);
    small += 2;
    s->launches_per_round = L.count + small;
    return PRL_OK;
}

// per-call block (Adam scalars of every round as torch evaluates them in double, target-update flags, decay, the
// query-alone switch, pointers), uploaded on `st`.  steps0 = the training-step count the reference's learn_batch sees in
// round 0; round r updates the target first when (steps0 + r + 1) % target_update_freq == 0.
static int duel_upload(prl_duel *s, int rounds, int64_t steps0, float *out_loss, const DuelCall &dense, cudaStream_t st) {
    const prl_duel_cfg &c = s->cfg;
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
    DuelCall *hc = reinterpret_cast<DuelCall *>(tail + duel_call_offset(MR));
    *hc = dense;
    hc->slots = s->slots; hc->out_loss = out_loss;
    hc->decay = (float)(1.0 - c.lr * c.weight_decay);
    *reinterpret_cast<int *>(hc + 1) = 0;
    PRL_CUDA(cudaMemcpyAsync(s->scal, tail, s->tail_bytes, cudaMemcpyHostToDevice, st));
    PRL_CUDA(cudaEventRecord(s->tail_done[sb], st));
    return PRL_OK;
}

static int duel_run(prl_duel *s, prl_buf *buf, int rounds, int batch, cudaStream_t st) {
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
                duel_round(s, buf, batch, cs);
                e = cudaStreamEndCapture(cs, &graph);
            }
            if (e == cudaSuccess) e = cudaGraphInstantiate(&s->graph_exec[g], graph, 0);
            if (graph) cudaGraphDestroy(graph);
            cudaStreamDestroy(cs);
            if (e != cudaSuccess) { s->graph_exec[g] = nullptr; return fail(PRL_ECUDA, "prl_duel: graph capture failed: %s", cudaGetErrorString(e)); }
            s->graph_batch[g] = batch;
            if (buf) { s->graph_buf = buf->records; s->graph_dynamic = dynamic; }
        }
        for (int r = 0; r < rounds; r++) PRL_CUDA(cudaGraphLaunch(s->graph_exec[g], st));
    } else {
        for (int r = 0; r < rounds; r++) {
            int rc = duel_round(s, buf, batch, st);
            if (rc) return rc;
        }
    }
    PRL_CUDA(cudaGetLastError());
    s->adam_step += rounds;
    s->last_launches = (int64_t)s->launches_per_round * rounds;
    return PRL_OK;
}

extern "C" int prl_duel_learn(prl_duel *s, prl_buf *buf, int rounds, int batch, int64_t training_steps, float *out_loss,
                              int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && out_loss, "null argument");
    const prl_duel_cfg &c = s->cfg;
    PRL_REQUIRE(rounds > 0 && rounds <= c.max_rounds && batch > 0 && batch <= c.max_batch, "rounds / batch outside the configured maxima");
    PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.obs_dim == c.obs_dim && buf->desc.n_actions == c.n_actions,
                "dueling DQN needs a discrete-action buffer with obs_dim = %d and n_actions = %d", c.obs_dim, c.n_actions);
    PRL_REQUIRE(buf->shard_world <= 1, "the buffer is one shard of a multi-GPU buffer: dueling DQN samples local buffers only");
    cudaStream_t st = (cudaStream_t)stream_;
    int rc = prl_buf_sample_indices(buf, rounds, batch, out_logical ? out_logical : s->logical, s->slots, stream_);
    if (rc) return rc;
    DuelCall dense;
    memset(&dense, 0, sizeof(dense));
    rc = duel_upload(s, rounds, training_steps + 1, out_loss, dense, st);   // PolicyLearner.learn counts the round first
    if (rc) return rc;
    return duel_run(s, buf, rounds, batch, st);
}

extern "C" int prl_duel_learn_batch(prl_duel *s, int batch, const float *state, const int32_t *action_id, const float *reward,
                                    const float *next_state, const uint8_t *terminated, const int32_t *curr_ids,
                                    const int32_t *next_ids, const uint8_t *next_unavailable, int64_t training_steps,
                                    float *out_loss, void *stream_) {
    PRL_REQUIRE(s && state && action_id && reward && next_state && terminated && out_loss, "null argument");
    PRL_REQUIRE(batch > 0 && batch <= s->cfg.max_batch, "batch outside the configured maximum");
    cudaStream_t st = (cudaStream_t)stream_;
    DuelCall dense;
    memset(&dense, 0, sizeof(dense));
    dense.d_state = state; dense.d_next_state = next_state; dense.d_reward = reward; dense.d_action_id = action_id;
    dense.d_curr_ids = curr_ids; dense.d_next_ids = next_ids; dense.d_next_unavail = next_unavailable; dense.d_term = terminated;
    dense.query_alone = curr_ids ? 0 : 1;
    int rc = duel_upload(s, 1, training_steps, out_loss, dense, st);
    if (rc) return rc;
    return duel_run(s, nullptr, 1, batch, st);
}

// Q(s, .) over an id set of K slots per row, the mean over that set: the forward of the round on n rows (chunks of
// max_batch rows through the workspace).  ids null: every action (K = n_actions).
extern "C" int prl_duel_q_values(prl_duel *s, int n, const float *state, const int32_t *ids, int K, int target, float *out_q, void *stream_) {
    PRL_REQUIRE(s && state && out_q, "null argument");
    const prl_duel_cfg &c = s->cfg;
    if (!ids) K = c.n_actions;
    PRL_REQUIRE(K >= 1 && K <= c.n_actions + 1, "the id set must hold 1 to %d slots per row", c.n_actions + 1);
    if (n <= 0) return PRL_OK;
    const float *w = target ? s->q_t : s->q;
    GemmLauncher L; L.st = (cudaStream_t)stream_;
    for (int r0 = 0; r0 < n; r0 += c.max_batch) {
        const int m = n - r0 < c.max_batch ? n - r0 : c.max_batch;
        duel_fwd(s, L, w, state + (size_t)r0 * c.obs_dim, m, K, ids ? ids + (size_t)r0 * K : nullptr, s->on);
        k_duel_q<<<(m * 32 + 127) / 128, 128, 0, L.st>>>(m, K, s->on.V, s->on.adv, out_q + (size_t)r0 * K);
    }
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

extern "C" int prl_duel_set_graph(prl_duel *s, int enable) {
    PRL_REQUIRE(s, "null handle");
    s->use_graph = enable != 0;
    return PRL_OK;
}
extern "C" int64_t prl_duel_last_launches(const prl_duel *s) { return s ? s->last_launches : -1; }
