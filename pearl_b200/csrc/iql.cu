// iql.cu — Implicit Q-Learning, Pearl's offline actor-critic (ImplicitQLearning.learn_batch, driven by PolicyLearner.learn
// or called directly on a caller's batch), replacing
//   policy_learners/sequential_decision_making/implicit_q_learning.py:159-302   learn_batch, _value_loss, _actor_loss,
//       _critic_loss, _expectile_loss
//   neural_networks/common/value_networks.py (VanillaValueNetwork), neural_networks/sequential_decision_making/
//       actor_networks.py (VanillaActorNetwork softmax; VanillaContinuousActorNetwork tanh + action_scaling)
//   utils/functional_utils/learning/critic_utils.py:170-203 (twin_critic_action_value_loss)
//
// One round: every loss from the parameters as they were before the round, then the value, critic and actor AdamW steps
// (three independent backward chains), then the critic soft update.  Fixed launch sequence, captured once per
// (batch, buffer) into a CUDA graph and replayed (DESIGN.md §3.4, as sac_discrete.cu).  The value net runs once over 2B
// rows (S' follows S in the workspace); the target critic at (s, a) serves both random picks.  Discrete actions enter the
// critic as the column W1[:, obs + a] (the one-hot fold).  The round's two random picks (torch.randint draws made by the
// caller) and every learning-rate-dependent scalar are read through the per-call block, so prl_iql_set_lr needs no new
// capture.  fp32, fixed summation order: bit-reproducible run to run.
#include <math.h>
#include <stdarg.h>

#include <new>

#include "common.cuh"
#include "gemm.cuh"

using namespace prl;

namespace {

// per-call block the captured round reads through
struct IqlCall {
    const int32_t *slots;                     // [rounds][B] (learn)
    const int32_t *bits;                      // [rounds][2]: target-critic pick of the value loss, then of the actor loss
    float *out_value, *out_critic, *out_actor;
    // learn_batch: the caller's dense batch
    const float *d_state, *d_next_state, *d_reward, *d_action;
    const int32_t *d_action_id;
    const uint8_t *d_term;
    float decay_a, decay_c, decay_v;          // AdamW decoupled decay 1 - lr * weight_decay (actor, critics, value)
};

// rows of one round: S [B][obs] with S' right after it (one 2B-row value pass), action id or continuous action, reward,
// terminated.  records == null: pack the caller's dense batch from the call block instead of gathering from the ring.
__global__ void k_iql_load(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int act_dim, const IqlCall *__restrict__ call,
                           const int *__restrict__ round_idx, int B, float *__restrict__ S, float *__restrict__ Act, int *__restrict__ act_id,
                           float *__restrict__ R, float *__restrict__ T) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    float *S2 = S + (size_t)B * obs;
    if (!records) {
        for (int p = lane; p < obs; p += 32) {
            S[(size_t)w * obs + p] = call->d_state[(size_t)w * obs + p];
            S2[(size_t)w * obs + p] = call->d_next_state[(size_t)w * obs + p];
        }
        for (int p = lane; p < act_dim; p += 32) Act[(size_t)w * act_dim + p] = call->d_action[(size_t)w * act_dim + p];
        if (lane == 0) {
            if (!act_dim) act_id[w] = call->d_action_id[w];
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
    for (int p = lane; p < act_dim; p += 32) Act[(size_t)w * act_dim + p] = __uint_as_float(r[L.off_action + p]);
    if (lane == 0) {
        if (!act_dim) act_id[w] = (int)r[L.off_action];
        R[w] = __uint_as_float(r[L.off_reward]);
        T[w] = (r[L.off_flags] & 1u) ? 1.f : 0.f;
    }
}

// The three losses of one round and the gradients they send into their networks (implicit_q_learning.py:159-286).
//   value : u = tq_v - V(s), w = expectile if u > 0 else 1 - expectile; L = mean(w u^2); dV = -2 w u / B
//   critic: y = V(s') gamma (1 - terminated) + r; L = (mean (q1 - y)^2 + mean (q2 - y)^2) / 2; dq_z = (q_z - y) / B
//   actor : adv = min(exp((tq_a - V(s)) temperature), clamp) (no lower clamp, no gradient);
//           discrete   L = -mean(adv log(softmax(logits)[a]))            -> dlogits
//           continuous L = mean(adv mean_d (mu - a)^2), mu = tanh-scaled -> d pre-tanh
// tq_v / tq_a = target critic q1 or q2 at (s, a), picked by the round's two bits.  One CTA, fixed order.
__global__ void __launch_bounds__(256) k_iql_losses(int B, int n_out, int discrete, const float *__restrict__ V, const float *__restrict__ qt,
                                                   const float *__restrict__ q, const float *__restrict__ R, const float *__restrict__ T,
                                                   const float *__restrict__ out, const int *__restrict__ act_id, const float *__restrict__ Act,
                                                   const float *__restrict__ low, const float *__restrict__ high, float gamma, float expectile,
                                                   float temperature, float clamp, float *__restrict__ dV, float *__restrict__ dq,
                                                   float *__restrict__ dout, const IqlCall *__restrict__ call, const int *__restrict__ round_idx) {
    __shared__ float red[3][256];
    const int rnd = *round_idx;
    const int pick_v = call->bits[2 * rnd], pick_a = call->bits[2 * rnd + 1];
    const float *tqv = qt + (pick_v ? B : 0), *tqa = qt + (pick_a ? B : 0);
    const float ib = 1.f / (float)B, id = 1.f / (float)n_out;
    float sv = 0.f, sc = 0.f, sa = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float vs = V[b];
        // value
        const float u = tqv[b] - vs, w = u > 0.f ? expectile : 1.f - expectile;
        sv += w * (u * u);
        dV[b] = -2.f * w * u * ib;
        // critic
        const float y = __fadd_rn(__fmul_rn(__fmul_rn(V[B + b], gamma), 1.f - T[b]), R[b]);
        const float e1 = q[b] - y, e2 = q[B + b] - y;
        sc += e1 * e1 + e2 * e2;
        dq[b] = e1 * ib;
        dq[B + b] = e2 * ib;
        // actor
        const float adv = fminf(expf((tqa[b] - vs) * temperature), clamp);
        const float *o = out + (size_t)b * n_out;
        float *g = dout + (size_t)b * n_out;
        if (discrete) {
            const RowSoftmax sm(o, n_out);
            const int a = act_id[b];
            sa -= adv * logf(sm(a));
            const float gb = -adv * ib;      // d L / d log p_a; softmax backward: g (onehot_a - p)
            for (int k = 0; k < n_out; k++) g[k] = gb * ((k == a ? 1.f : 0.f) - sm(k));
        } else {
            float l = 0.f;
            for (int d = 0; d < n_out; d++) {
                const float lo = low[d], hi = high[d], t = tanhf(o[d]);
                const float mu = (((hi - lo) * (t + 1.0f)) / 2.f) + lo;
                const float df = mu - Act[(size_t)b * n_out + d];
                l += df * df;
                g[d] = adv * ib * id * 2.f * df * ((hi - lo) * 0.5f) * (1.f - t * t);
            }
            sa += adv * (l * id);
        }
    }
    red[0][threadIdx.x] = sv; red[1][threadIdx.x] = sc; red[2][threadIdx.x] = sa;
    __syncthreads();
    for (int o = 128; o; o >>= 1) {
        if (threadIdx.x < o)
            for (int k = 0; k < 3; k++) red[k][threadIdx.x] += red[k][threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        call->out_value[rnd] = red[0][0] * ib;
        call->out_critic[rnd] = red[1][0] * ib * 0.5f;
        call->out_actor[rnd] = red[2][0] * ib;
    }
}

__global__ void k_iql_bump(int *round_idx) { *round_idx += 1; }

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_iql {
    prl_iql_cfg cfg;
    int Pa, Pc, Pv;
    int aW1, ab1, aW2, ab2, aW3, ab3;
    int cW1, cb1, cW2, cb2, cW3, cb3;
    int vW1, vb1, vW2, vb2, vW3, vb3;
    float *actor, *actor_m, *actor_v, *actor_x;
    float *critic, *critic_m, *critic_v, *critic_x, *critic_t;
    float *value, *value_m, *value_v, *value_x;
    const float *low, *high;
    int64_t adam_step;
    // workspace
    float *S, *Act, *R, *T, *v1, *v2, *V, *P, *c1t, *c2t, *qt, *c1, *c2, *q, *h1, *h2, *out, *dout, *dV, *dv2, *dv1, *dq, *dc2, *dc1,
        *dh2, *dh1, *g_actor, *g_critic, *g_value;
    int *act;
    int32_t *slots, *logical;
    float2 *scal_a, *scal_c, *scal_v;
    IqlCall *call;
    int *round_idx;
    bool use_graph;
    cudaGraphExec_t graph_exec[2];            // [0] rounds from a replay buffer, [1] learn_batch on a dense batch
    int graph_batch[2];
    const uint32_t *graph_buf;
    int launches_per_round;
    float2 *scal_host[2];
    cudaEvent_t scal_done[2];
    int scal_next;
    int64_t last_launches;
};

static int64_t al64(int64_t x) { return (x + 255) / 256 * 256; }

static bool iql_discrete(const prl_iql_cfg &c) { return c.n_actions > 0; }

static void iql_layout(prl_iql *s) {
    const prl_iql_cfg &c = s->cfg;
    const int nout = iql_discrete(c) ? c.n_actions : c.act_dim;
    int o = 0;
    s->aW1 = o; o += c.actor_h1 * c.obs_dim; s->ab1 = o; o += c.actor_h1;
    s->aW2 = o; o += c.actor_h2 * c.actor_h1; s->ab2 = o; o += c.actor_h2;
    s->aW3 = o; o += nout * c.actor_h2; s->ab3 = o; o += nout;
    s->Pa = o;
    const int D = c.obs_dim + nout;
    o = 0;
    s->cW1 = o; o += c.critic_h1 * D; s->cb1 = o; o += c.critic_h1;
    s->cW2 = o; o += c.critic_h2 * c.critic_h1; s->cb2 = o; o += c.critic_h2;
    s->cW3 = o; o += c.critic_h2; s->cb3 = o; o += 1;
    s->Pc = o;
    o = 0;
    s->vW1 = o; o += c.value_h1 * c.obs_dim; s->vb1 = o; o += c.value_h1;
    s->vW2 = o; o += c.value_h2 * c.value_h1; s->vb2 = o; o += c.value_h2;
    s->vW3 = o; o += c.value_h2; s->vb3 = o; o += 1;
    s->Pv = o;
}

static int iql_check(const prl_iql_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->actor_h1 > 0 && c->actor_h2 > 0 && c->critic_h1 > 0 && c->critic_h2 > 0 && c->value_h1 > 0 &&
                    c->value_h2 > 0, "dimensions must be positive");
    PRL_REQUIRE((c->n_actions > 0) != (c->act_dim > 0) && c->n_actions >= 0 && c->act_dim >= 0,
                "exactly one of n_actions (discrete) and act_dim (continuous) must be positive");
    PRL_REQUIRE(c->n_actions <= 255, "n_actions must be in [1, 255]");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    return PRL_OK;
}

extern "C" int64_t prl_iql_actor_param_count(const prl_iql_cfg *c) {
    if (iql_check(c)) return -1;
    prl_iql t; t.cfg = *c; iql_layout(&t);
    return t.Pa;
}
extern "C" int64_t prl_iql_critic_param_count(const prl_iql_cfg *c) {
    if (iql_check(c)) return -1;
    prl_iql t; t.cfg = *c; iql_layout(&t);
    return t.Pc;
}
extern "C" int64_t prl_iql_value_param_count(const prl_iql_cfg *c) {
    if (iql_check(c)) return -1;
    prl_iql t; t.cfg = *c; iql_layout(&t);
    return t.Pv;
}

struct IqlWs { int64_t off[40]; int64_t total; };
static IqlWs iql_ws(const prl_iql_cfg *c, int Pa, int Pc, int Pv) {
    IqlWs w; int64_t o = 0; int k = 0;
    const int64_t B = c->max_batch, O = c->obs_dim, N = iql_discrete(*c) ? c->n_actions : c->act_dim;
    const int64_t C1 = c->critic_h1, C2 = c->critic_h2;
    auto add = [&](int64_t words) { w.off[k++] = o; o = al64(o + words * 4); };
    add(2 * B * O); add(B * (c->act_dim > 0 ? c->act_dim : 1)); add(B); add(B);                  // S|S' Act R T
    add(2 * B * c->value_h1); add(2 * B * c->value_h2); add(2 * B);                              // v1 v2 V
    add(2 * B * C1); add(2 * B * C1); add(2 * B * C2); add(2 * B);                               // P c1t c2t qt
    add(2 * B * C1); add(2 * B * C2); add(2 * B);                                                // c1 c2 q
    add(B * c->actor_h1); add(B * c->actor_h2); add(B * N); add(B * N);                          // h1 h2 out dout
    add(B); add(B * c->value_h2); add(B * c->value_h1);                                          // dV dv2 dv1
    add(2 * B); add(2 * B * C2); add(2 * B * C1);                                                // dq dc2 dc1
    add(B * c->actor_h2); add(B * c->actor_h1);                                                  // dh2 dh1
    add(Pa); add(2 * (int64_t)Pc); add(Pv);                                                      // g_actor g_critic g_value
    add(B);                                                                                      // act (int32)
    add((int64_t)c->max_rounds * B); add((int64_t)c->max_rounds * B);                           // slots logical (int32)
    add(6 * (int64_t)c->max_rounds + 64);                                                        // scal_a | scal_c | scal_v | call | round_idx
    w.total = o;
    return w;
}
extern "C" int64_t prl_iql_workspace_bytes(const prl_iql_cfg *c) {
    if (iql_check(c)) return -1;
    prl_iql t; t.cfg = *c; iql_layout(&t);
    return iql_ws(c, t.Pa, t.Pc, t.Pv).total;
}

extern "C" int prl_iql_create(prl_iql **out, const prl_iql_cfg *cfg, float *actor_w, float *actor_m, float *actor_v, float *actor_vmax,
                              float *critic_w, float *critic_m, float *critic_v, float *critic_vmax, float *critic_target_w,
                              float *value_w, float *value_m, float *value_v, float *value_vmax, const float *low_dev,
                              const float *high_dev, int64_t adam_step, void *workspace) {
    PRL_REQUIRE(out && actor_w && actor_m && actor_v && actor_vmax && critic_w && critic_m && critic_v && critic_vmax && critic_target_w &&
                    value_w && value_m && value_v && value_vmax && workspace, "null argument");
    int rc = iql_check(cfg);
    if (rc) return rc;
    PRL_REQUIRE(iql_discrete(*cfg) || (low_dev && high_dev), "continuous actions need the action box (low / high)");
    prl_iql *s = new (std::nothrow) prl_iql();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    iql_layout(s);
    s->actor = actor_w; s->actor_m = actor_m; s->actor_v = actor_v; s->actor_x = actor_vmax;
    s->critic = critic_w; s->critic_m = critic_m; s->critic_v = critic_v; s->critic_x = critic_vmax; s->critic_t = critic_target_w;
    s->value = value_w; s->value_m = value_m; s->value_v = value_v; s->value_x = value_vmax;
    s->low = low_dev; s->high = high_dev;
    s->adam_step = adam_step;
    IqlWs w = iql_ws(cfg, s->Pa, s->Pc, s->Pv);
    char *b = (char *)workspace;
    float **f[] = {&s->S, &s->Act, &s->R, &s->T, &s->v1, &s->v2, &s->V, &s->P, &s->c1t, &s->c2t, &s->qt, &s->c1, &s->c2, &s->q, &s->h1,
                   &s->h2, &s->out, &s->dout, &s->dV, &s->dv2, &s->dv1, &s->dq, &s->dc2, &s->dc1, &s->dh2, &s->dh1, &s->g_actor,
                   &s->g_critic, &s->g_value};
    int k = 0;
    for (auto p : f) *p = (float *)(b + w.off[k++]);
    s->act = (int *)(b + w.off[k++]);
    s->slots = (int32_t *)(b + w.off[k++]); s->logical = (int32_t *)(b + w.off[k++]);
    s->scal_a = (float2 *)(b + w.off[k++]); s->scal_c = s->scal_a + cfg->max_rounds; s->scal_v = s->scal_c + cfg->max_rounds;
    s->call = (IqlCall *)(s->scal_v + cfg->max_rounds); s->round_idx = (int *)(s->call + 1);
    static_assert(sizeof(IqlCall) + 4 <= 64 * 4, "call block fits the reserved tail");
    s->scal_next = 0; s->use_graph = true; s->graph_exec[0] = s->graph_exec[1] = nullptr; s->graph_batch[0] = s->graph_batch[1] = 0;
    s->graph_buf = nullptr; s->last_launches = 0; s->launches_per_round = 0;
    cudaError_t e = cudaSuccess;
    int made = 0;   // pinned buffer / event pairs fully created
    s->scal_host[0] = s->scal_host[1] = nullptr;
    for (int i = 0; i < 2 && e == cudaSuccess; i++) {
        e = cudaHostAlloc((void **)&s->scal_host[i], (size_t)cfg->max_rounds * 24 + 256, cudaHostAllocDefault);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->scal_done[i], cudaEventDisableTiming);
        if (e == cudaSuccess) made++;
    }
    if (e != cudaSuccess) {
        for (int i = 0; i < made; i++) { cudaEventDestroy(s->scal_done[i]); cudaFreeHost(s->scal_host[i]); }
        if (made < 2 && s->scal_host[made]) cudaFreeHost(s->scal_host[made]);   // its event was not created
        delete s;
        return fail(PRL_ECUDA, "prl_iql_create: %s", cudaGetErrorString(e));
    }
    *out = s;
    return PRL_OK;
}
extern "C" int prl_iql_destroy(prl_iql *s) {
    if (!s) return PRL_OK;
    for (int i = 0; i < 2; i++) { cudaEventSynchronize(s->scal_done[i]); cudaEventDestroy(s->scal_done[i]); cudaFreeHost(s->scal_host[i]); }
    for (int i = 0; i < 2; i++) if (s->graph_exec[i]) cudaGraphExecDestroy(s->graph_exec[i]);
    delete s;
    return PRL_OK;
}
extern "C" int64_t prl_iql_adam_step(const prl_iql *s) { return s ? s->adam_step : -1; }

extern "C" int prl_iql_set_lr(prl_iql *s, double actor_lr, double critic_lr, double value_lr) {
    PRL_REQUIRE(s, "null handle");
    PRL_REQUIRE(actor_lr >= 0.0 && critic_lr >= 0.0 && value_lr >= 0.0, "learning rates must be non-negative");
    s->cfg.actor_lr = actor_lr;
    s->cfg.critic_lr = critic_lr;
    s->cfg.value_lr = value_lr;
    return PRL_OK;
}

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
static int iql_round(prl_iql *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_iql_cfg &c = s->cfg;
    const bool disc = iql_discrete(c);
    const int O = c.obs_dim, N = disc ? c.n_actions : c.act_dim, D = O + N;
    const int H1 = c.actor_h1, H2 = c.actor_h2, C1 = c.critic_h1, C2 = c.critic_h2, V1 = c.value_h1, V2 = c.value_h2;
    const long long Pc = s->Pc;
    // the decay factors are overridden by call->decay_a / decay_c / decay_v (k_adamw's decay pointer)
    const AdamHp h = adam_hp(0.0, c.beta1, c.beta2, c.eps, c.weight_decay);
    GemmLauncher L; L.st = st;
    const float *aw = s->actor, *cw = s->critic, *vw = s->value;
    const long long sC1 = (long long)B * C1, sC2 = (long long)B * C2;
    const int eb = 256;
    int small = 0;
    float *S = s->S;
    // critic q1, q2 at (s, a): the action as the one-hot fold (discrete) or as the second half of the input (continuous)
    auto critic_sa = [&](const float *net, float *c1, float *c2, float *q) {
        if (disc) {
            L.fwd(mat(S, O), B, net + s->cW1, D, Pc, net + s->cb1, Pc, C1, O, false, s->P, C1, sC1, 2);
            k_fold<<<dim3((B * C1 + eb - 1) / eb, 1, 2), eb, 0, st>>>(B, C1, s->P, net + s->cW1 + O, D, Pc, s->act, c1);
            small++;
        } else {
            L.fwd(mat2(S, O, O, s->Act, N), B, net + s->cW1, D, Pc, net + s->cb1, Pc, C1, D, true, c1, C1, sC1, 2);
        }
        L.fwd(mat(c1, C1, sC1), B, net + s->cW2, C1, Pc, net + s->cb2, Pc, C2, C1, true, c2, C2, sC2, 2);
        L.fwd(mat(c2, C2, sC2), B, net + s->cW3, C2, Pc, net + s->cb3, Pc, 1, C2, false, q, 1, B, 2);
    };
    k_iql_load<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf ? buf->records : nullptr, buf ? buf->lay : prl_buf_layout{}, O, disc ? 0 : N,
                                                     s->call, s->round_idx, B, S, s->Act, s->act, s->R, s->T);
    small++;
    // ---------------- forward passes, all from the pre-round parameters
    L.fwd(mat(S, O), 2 * B, vw + s->vW1, O, 0, vw + s->vb1, 0, V1, O, true, s->v1, V1, 0);            // V(s) | V(s')
    L.fwd(mat(s->v1, V1), 2 * B, vw + s->vW2, V1, 0, vw + s->vb2, 0, V2, V1, true, s->v2, V2, 0);
    L.fwd(mat(s->v2, V2), 2 * B, vw + s->vW3, V2, 0, vw + s->vb3, 0, 1, V2, false, s->V, 1, 0);
    critic_sa(s->critic_t, s->c1t, s->c2t, s->qt);                                                      // target critic
    critic_sa(cw, s->c1, s->c2, s->q);                                                                  // online critic
    L.fwd(mat(S, O), B, aw + s->aW1, O, 0, aw + s->ab1, 0, H1, O, true, s->h1, H1, 0);                 // actor
    L.fwd(mat(s->h1, H1), B, aw + s->aW2, H1, 0, aw + s->ab2, 0, H2, H1, true, s->h2, H2, 0);
    L.fwd(mat(s->h2, H2), B, aw + s->aW3, H2, 0, aw + s->ab3, 0, N, H2, false, s->out, N, 0);
    k_iql_losses<<<1, 256, 0, st>>>(B, N, disc ? 1 : 0, s->V, s->qt, s->q, s->R, s->T, s->out, s->act, s->Act, s->low, s->high,
                                     (float)c.gamma, (float)c.expectile, (float)c.temperature, (float)c.advantage_clamp, s->dV, s->dq,
                                     s->dout, s->call, s->round_idx);
    small++;
    // ---------------- value step (expectile regression)
    {
        float *gv = s->g_value;
        L.bwd_w(s->dV, 1, 0, B, 1, mat(s->v2, V2), V2, gv + s->vW3, V2, 0, gv + s->vb3, 0);
        k_head_bwd<<<dim3((B * V2 + eb - 1) / eb, 1, 1), eb, 0, st>>>(B, V2, s->dV, vw + s->vW3, 0, s->v2, s->dv2);
        L.bwd_w(s->dv2, V2, 0, B, V2, mat(s->v1, V1), V1, gv + s->vW2, V1, 0, gv + s->vb2, 0);
        L.bwd_x(s->dv2, V2, 0, B, V2, vw + s->vW2, V1, 0, 0, V1, s->dv1, V1, 0, s->v1, V1, 0, false);
        L.bwd_w(s->dv1, V1, 0, B, V1, mat(S, O), O, gv + s->vW1, O, 0, gv + s->vb1, 0);
        k_adamw<<<(s->Pv + eb - 1) / eb, eb, 0, st>>>(s->Pv, s->value, s->value_m, s->value_v, s->value_x, gv, h, s->scal_v, s->round_idx,
                                                    nullptr, 0.f, 0.f, &s->call->decay_v);
        small += 2;
    }
    // ---------------- critic step (twin MSE against r + gamma V(s')) and soft update of the targets with the new parameters
    {
        float *gc = s->g_critic;
        L.bwd_w(s->dq, 1, B, B, 1, mat(s->c2, C2, sC2), C2, gc + s->cW3, C2, Pc, gc + s->cb3, Pc, 2);
        k_head_bwd<<<dim3((B * C2 + eb - 1) / eb, 1, 2), eb, 0, st>>>(B, C2, s->dq, cw + s->cW3, Pc, s->c2, s->dc2);
        L.bwd_w(s->dc2, C2, sC2, B, C2, mat(s->c1, C1, sC1), C1, gc + s->cW2, C1, Pc, gc + s->cb2, Pc, 2);
        L.bwd_x(s->dc2, C2, sC2, B, C2, cw + s->cW2, C1, Pc, 0, C1, s->dc1, C1, sC1, s->c1, C1, sC1, false, 2);
        if (disc) {
            L.bwd_w(s->dc1, C1, sC1, B, C1, mat(S, O), O, gc + s->cW1, D, Pc, gc + s->cb1, Pc, 2);   // state columns + b1
            k_fold_w1a_grad<<<dim3((C1 * N + eb - 1) / eb, 1, 2), eb, 0, st>>>(B, N, C1, s->act, s->dc1, gc + s->cW1 + O, D, Pc);
            small++;
        } else {
            L.bwd_w(s->dc1, C1, sC1, B, C1, mat2(S, O, O, s->Act, N), D, gc + s->cW1, D, Pc, gc + s->cb1, Pc, 2);
        }
        const int n2p = 2 * s->Pc;
        k_adamw<<<(n2p + eb - 1) / eb, eb, 0, st>>>(n2p, s->critic, s->critic_m, s->critic_v, s->critic_x, gc, h, s->scal_c, s->round_idx,
                                                  s->critic_t, (float)c.tau, (float)(1.0 - c.tau), &s->call->decay_c);
        small += 2;
    }
    // ---------------- actor step (advantage-weighted regression)
    {
        float *ga = s->g_actor;
        L.bwd_w(s->dout, N, 0, B, N, mat(s->h2, H2), H2, ga + s->aW3, H2, 0, ga + s->ab3, 0);
        L.bwd_x(s->dout, N, 0, B, N, aw + s->aW3, H2, 0, 0, H2, s->dh2, H2, 0, s->h2, H2, 0, false);
        L.bwd_w(s->dh2, H2, 0, B, H2, mat(s->h1, H1), H1, ga + s->aW2, H1, 0, ga + s->ab2, 0);
        L.bwd_x(s->dh2, H2, 0, B, H2, aw + s->aW2, H1, 0, 0, H1, s->dh1, H1, 0, s->h1, H1, 0, false);
        L.bwd_w(s->dh1, H1, 0, B, H1, mat(S, O), O, ga + s->aW1, O, 0, ga + s->ab1, 0);
        k_adamw<<<(s->Pa + eb - 1) / eb, eb, 0, st>>>(s->Pa, s->actor, s->actor_m, s->actor_v, s->actor_x, ga, h, s->scal_a, s->round_idx,
                                                    nullptr, 0.f, 0.f, &s->call->decay_a);
        small++;
    }
    k_iql_bump<<<1, 1, 0, st>>>(s->round_idx);
    small++;
    s->launches_per_round = L.count + small;
    return PRL_OK;
}

// per-call block (Adam scalars of every round as torch evaluates them in double, decay factors, pointers), uploaded on `st`
static int iql_upload(prl_iql *s, int rounds, const int32_t *bits, float *out_value, float *out_critic, float *out_actor, const IqlCall &dense,
                      cudaStream_t st) {
    const prl_iql_cfg &c = s->cfg;
    const int sb = s->scal_next; s->scal_next ^= 1;
    PRL_CUDA(cudaEventSynchronize(s->scal_done[sb]));
    float2 *hs = s->scal_host[sb];
    const int MR = c.max_rounds;
    for (int r = 0; r < rounds; r++) {
        const double step = (double)(s->adam_step + r + 1);
        const double bc1 = 1.0 - pow(c.beta1, step), bc2 = 1.0 - pow(c.beta2, step);
        hs[r] = make_float2((float)(c.actor_lr / bc1), (float)sqrt(bc2));
        hs[MR + r] = make_float2((float)(c.critic_lr / bc1), (float)sqrt(bc2));
        hs[2 * MR + r] = make_float2((float)(c.value_lr / bc1), (float)sqrt(bc2));
    }
    IqlCall *hc = reinterpret_cast<IqlCall *>(hs + 3 * (size_t)MR);
    *hc = dense;
    hc->slots = s->slots; hc->bits = bits; hc->out_value = out_value; hc->out_critic = out_critic; hc->out_actor = out_actor;
    hc->decay_a = (float)(1.0 - c.actor_lr * c.weight_decay);
    hc->decay_c = (float)(1.0 - c.critic_lr * c.weight_decay);
    hc->decay_v = (float)(1.0 - c.value_lr * c.weight_decay);
    *reinterpret_cast<int *>(hc + 1) = 0;
    // scal_a | scal_c | scal_v | call | round_idx are contiguous on the device in the same order
    PRL_CUDA(cudaMemcpyAsync(s->scal_a, hs, 3 * (size_t)MR * 8 + sizeof(IqlCall) + 4, cudaMemcpyHostToDevice, st));
    PRL_CUDA(cudaEventRecord(s->scal_done[sb], st));
    return PRL_OK;
}

static int iql_run(prl_iql *s, prl_buf *buf, int rounds, int batch, cudaStream_t st) {
    const int g = buf ? 0 : 1;
    if (s->use_graph) {
        if (!s->graph_exec[g] || s->graph_batch[g] != batch || (buf && s->graph_buf != buf->records)) {
            if (s->graph_exec[g]) { cudaGraphExecDestroy(s->graph_exec[g]); s->graph_exec[g] = nullptr; }
            cudaStream_t cs;
            PRL_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
            cudaGraph_t graph = nullptr;
            cudaError_t e = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
            if (e == cudaSuccess) {
                iql_round(s, buf, batch, cs);
                e = cudaStreamEndCapture(cs, &graph);
            }
            if (e == cudaSuccess) e = cudaGraphInstantiate(&s->graph_exec[g], graph, 0);
            if (graph) cudaGraphDestroy(graph);
            cudaStreamDestroy(cs);
            if (e != cudaSuccess) { s->graph_exec[g] = nullptr; return fail(PRL_ECUDA, "prl_iql: graph capture failed: %s", cudaGetErrorString(e)); }
            s->graph_batch[g] = batch;
            if (buf) s->graph_buf = buf->records;
        }
        for (int r = 0; r < rounds; r++) PRL_CUDA(cudaGraphLaunch(s->graph_exec[g], st));
    } else {
        for (int r = 0; r < rounds; r++) {
            int rc = iql_round(s, buf, batch, st);
            if (rc) return rc;
        }
    }
    PRL_CUDA(cudaGetLastError());
    s->adam_step += rounds;
    s->last_launches = (int64_t)s->launches_per_round * rounds;
    return PRL_OK;
}

extern "C" int prl_iql_learn(prl_iql *s, prl_buf *buf, int rounds, int batch, const int32_t *bits_dev, float *out_value_loss,
                             float *out_critic_loss, float *out_actor_loss, int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && bits_dev && out_value_loss && out_critic_loss && out_actor_loss, "null argument");
    const prl_iql_cfg &c = s->cfg;
    PRL_REQUIRE(rounds > 0 && rounds <= c.max_rounds && batch > 0 && batch <= c.max_batch, "rounds / batch outside the configured maxima");
    PRL_REQUIRE(buf->desc.obs_dim == c.obs_dim, "IQL: the buffer's obs_dim (%d) is not the configured %d", buf->desc.obs_dim, c.obs_dim);
    if (iql_discrete(c))
        PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.n_actions == c.n_actions,
                    "IQL with discrete actions needs a discrete-action buffer with n_actions = %d", c.n_actions);
    else
        PRL_REQUIRE((buf->desc.flags & PRL_BUF_CONTINUOUS) && buf->desc.act_dim == c.act_dim,
                    "IQL with continuous actions needs a continuous-action buffer with act_dim = %d", c.act_dim);
    PRL_REQUIRE(buf->shard_world <= 1, "the buffer is one shard of a multi-GPU buffer: IQL samples local buffers only");
    cudaStream_t st = (cudaStream_t)stream_;
    int rc = prl_buf_sample_indices(buf, rounds, batch, out_logical ? out_logical : s->logical, s->slots, stream_);
    if (rc) return rc;
    IqlCall dense;
    memset(&dense, 0, sizeof(dense));
    rc = iql_upload(s, rounds, bits_dev, out_value_loss, out_critic_loss, out_actor_loss, dense, st);
    if (rc) return rc;
    return iql_run(s, buf, rounds, batch, st);
}

extern "C" int prl_iql_learn_batch(prl_iql *s, int batch, const float *state, const float *action, const int32_t *action_id,
                                   const float *reward, const float *next_state, const uint8_t *terminated, const int32_t *bits_dev,
                                   float *out_value_loss, float *out_critic_loss, float *out_actor_loss, void *stream_) {
    PRL_REQUIRE(s && state && reward && next_state && terminated && bits_dev && out_value_loss && out_critic_loss && out_actor_loss,
                "null argument");
    const prl_iql_cfg &c = s->cfg;
    PRL_REQUIRE(batch > 0 && batch <= c.max_batch, "batch outside the configured maximum");
    PRL_REQUIRE(iql_discrete(c) ? action_id != nullptr : action != nullptr,
                "discrete IQL takes action ids, continuous IQL takes continuous actions");
    cudaStream_t st = (cudaStream_t)stream_;
    IqlCall dense;
    memset(&dense, 0, sizeof(dense));
    dense.d_state = state; dense.d_next_state = next_state; dense.d_reward = reward; dense.d_action = action;
    dense.d_action_id = action_id; dense.d_term = terminated;
    int rc = iql_upload(s, 1, bits_dev, out_value_loss, out_critic_loss, out_actor_loss, dense, st);
    if (rc) return rc;
    return iql_run(s, nullptr, 1, batch, st);
}

extern "C" int prl_iql_set_graph(prl_iql *s, int enable) {
    PRL_REQUIRE(s, "null handle");
    s->use_graph = enable != 0;
    return PRL_OK;
}
extern "C" int64_t prl_iql_last_launches(const prl_iql *s) { return s ? s->last_launches : -1; }
