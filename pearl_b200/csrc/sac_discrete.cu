// sac_discrete.cu — discrete-action Soft Actor-Critic learner (SoftActorCritic.learn_batch driven by
// PolicyLearner.learn), replacing
//   policy_learners/sequential_decision_making/actor_critic_base.py:309-366   (actor step, critic step, soft update)
//   policy_learners/sequential_decision_making/soft_actor_critic.py            (learn_batch: entropy autotune with
//       torch.optim.Adam(eps=1e-4); _actor_loss; _critic_loss; _get_next_state_expected_values)
//   neural_networks/sequential_decision_making/actor_networks.py (VanillaActorNetwork: MLP + softmax)
//   neural_networks/sequential_decision_making/twin_critic.py, q_value_networks.py (get_q_values over all actions)
//   utils/functional_utils/learning/critic_utils.py (twin_critic_action_value_loss, update_critic_target_network)
//
// One round is the fixed launch sequence below, captured once per (batch, buffer) into a CUDA graph and replayed
// (DESIGN.md §3.4, as sac.cu).  Dense work goes through GemmLauncher.  The critic's one-hot action input is folded: the
// layer-1 state product is computed once per (row, critic) and the action enters as the column W1[:, obs + id] (the fold
// dqn.cu uses), so the all-action evaluation costs one B-row product plus B*A-row products for layers 2 and 3.  Every
// learning-rate-dependent scalar lives in the per-call block, so prl_sacd_set_lr needs no new capture.  fp32, fixed
// summation order: bit-reproducible run to run.
#include <math.h>
#include <stdarg.h>

#include <new>

#include "common.cuh"
#include "gemm.cuh"

using namespace prl;

namespace {

// per-call block the captured round reads through
struct SacdCall {
    const int32_t *slots;                 // [rounds][B]
    float *out_actor, *out_critic, *out_entropy;
    float decay_a, decay_c;               // AdamW decoupled decay 1 - lr * weight_decay (actor, critics)
};

// batch rows of one round: state, next state, action id, reward, terminated, and the next-action ids of every slot
// (slot k holds id_k; slots at and beyond the row's count are masked by k_sacd_target)
__global__ void k_sacd_gather(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int A, int dynamic,
                              const SacdCall *__restrict__ call, const int *__restrict__ round_idx, int B, float *__restrict__ S,
                              float *__restrict__ S2, int *__restrict__ act, float *__restrict__ R, float *__restrict__ T,
                              int *__restrict__ cnt, int *__restrict__ ids) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
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

// rows of the taken action: c1a[z][b] = c1[z][b*A + a_b] (and c2a, qa); the online critic does not change between the
// actor step and the critic step, so Q(s, a) and its activations are those of the all-action pass
__global__ void k_sacd_pick(int B, int A, int C1, int C2, const int *__restrict__ act, const float *__restrict__ c1, const float *__restrict__ c2,
                            const float *__restrict__ q, float *__restrict__ c1a, float *__restrict__ c2a, float *__restrict__ qa) {
    const int z = blockIdx.z, b = blockIdx.x;
    const size_t src = (size_t)b * A + act[b];
    if (threadIdx.x == 0) qa[z * B + b] = q[(size_t)z * B * A + src];
    for (int j = threadIdx.x; j < C1; j += blockDim.x) c1a[((size_t)z * B + b) * C1 + j] = c1[((size_t)z * B * A + src) * C1 + j];
    for (int j = threadIdx.x; j < C2; j += blockDim.x) c2a[((size_t)z * B + b) * C2 + j] = c2[((size_t)z * B * A + src) * C2 + j];
}

constexpr int kMaxA = 255;

// actor loss (soft_actor_critic.py _actor_loss): pi = softmax, q = min(Q1, Q2) over every action (current action sets are
// complete: nothing is masked), L = mean over B*A of pi * (alpha * log(pi + 1e-8) - q).  Writes dL/dlogits and, for the
// entropy step, sum_k pi * log(pi + 1e-8) per row of this (pre-update) actor.  One CTA, fixed order.
__global__ void __launch_bounds__(256) k_sacd_actor(int B, int A, const float *__restrict__ logits, const float *__restrict__ q,
                                                   const float *__restrict__ alpha, float *__restrict__ dlogit, float *__restrict__ ent,
                                                   const SacdCall *__restrict__ call, const int *__restrict__ round_idx) {
    __shared__ float red[256];
    const float al = *alpha, inv = 1.f / (float)(B * A);
    float s = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const RowSoftmax sm(logits + (size_t)b * A, A);
        // dL/dpi_k = (alpha log(pi_k + 1e-8) + alpha pi_k / (pi_k + 1e-8) - q_k) / (B A)
        auto grad_pi = [&](int k, float p, float lp) {
            const size_t o = (size_t)b * A + k;
            const float qk = fminf(q[o], q[(size_t)B * A + o]);
            return (al * lp + al * p / (p + 1e-8f) - qk) * inv;
        };
        float e = 0.f, dot = 0.f;
        for (int k = 0; k < A; k++) {
            const size_t o = (size_t)b * A + k;
            const float p = sm(k), lp = logf(p + 1e-8f);
            s += p * (al * lp - fminf(q[o], q[(size_t)B * A + o]));
            e += p * lp;
            dot += p * grad_pi(k, p, lp);
        }
        for (int k = 0; k < A; k++) {   // softmax backward
            const float p = sm(k);
            dlogit[(size_t)b * A + k] = p * (grad_pi(k, p, logf(p + 1e-8f)) - dot);
        }
        ent[b] = e;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) call->out_actor[*round_idx] = red[0] * inv;
}

// critic target (_get_next_state_expected_values, _critic_loss): q~_k = min(Q1t, Q2t)(s', one-hot(id_k)), 0 on masked slots;
// V = sum over ALL A slots of pi'_k (q~_k - alpha log(pi'_k + 1e-8)), pi' the UPDATED actor's output k;
// y = V * gamma * (1 - terminated) + reward
__global__ void k_sacd_target(int B, int A, const float *__restrict__ logits, const float *__restrict__ qt, const int *__restrict__ cnt,
                              const float *__restrict__ alpha, float gamma, const float *__restrict__ term, const float *__restrict__ rew,
                              float *__restrict__ y) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const RowSoftmax sm(logits + (size_t)b * A, A);
    const float al = *alpha;
    float v = 0.f;
    for (int k = 0; k < A; k++) {
        const size_t o = (size_t)b * A + k;
        const float p = sm(k);
        const float qk = k < cnt[b] ? fminf(qt[o], qt[(size_t)B * A + o]) : 0.f;
        v += (qk - al * logf(p + 1e-8f)) * p;
    }
    y[b] = __fadd_rn(__fmul_rn(__fmul_rn(v, gamma), 1.f - term[b]), rew[b]);
}

// (MSE(Q1(s,a), y) + MSE(Q2(s,a), y)) / 2 with qa = Q(s, a) picked from the all-action pass; dq_z = (q_z - y) / B
__global__ void __launch_bounds__(256) k_sacd_critic_loss(int B, const float *__restrict__ qa,
                                                         const float *__restrict__ y, float *__restrict__ dq, const SacdCall *__restrict__ call,
                                                         const int *__restrict__ round_idx) {
    __shared__ float red[256];
    float s = 0.f;
    const float ib = 1.f / (float)B;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float e1 = qa[b] - y[b], e2 = qa[B + b] - y[b];
        s += e1 * e1 + e2 * e2;
        dq[b] = e1 * ib;
        dq[B + b] = e2 * ib;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) call->out_critic[*round_idx] = red[0] * ib * 0.5f;
}

// entropy step (soft_actor_critic.py learn_batch): H = -mean_b sum_k pi log(pi + 1e-8) of the actor-step probabilities;
// loss = exp(log_alpha) (H - target_entropy); torch.optim.Adam (no weight decay, no amsgrad) on log_alpha; alpha = exp.
// Also advances the round counter.  One thread does the arithmetic.
__global__ void __launch_bounds__(256) k_sacd_alpha(int B, const float *__restrict__ ent, float target_entropy, float *__restrict__ la /* [3]: w m v */,
                                                   float *__restrict__ alpha, float omb1, float beta2, float omb2, float eps,
                                                   const float2 *__restrict__ scal, const int *__restrict__ round_idx,
                                                   const SacdCall *__restrict__ call, int autotune) {
    __shared__ float red[256];
    if (!autotune) {
        if (threadIdx.x == 0) *const_cast<int *>(round_idx) += 1;
        return;
    }
    float s = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) s += ent[b];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) {
        const float H = -(red[0] / (float)B);
        const float g = expf(la[0]) * (H - target_entropy);   // the loss; also d loss / d log_alpha
        call->out_entropy[*round_idx] = g;
        const float2 sc = scal[*round_idx];
        float m = la[1], v = la[2];
        m = fmaf(omb1, g - m, m);
        v = __fadd_rn(__fmul_rn(v, beta2), __fmul_rn(__fmul_rn(omb2, g), g));
        const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), sc.y), eps);
        const float p = __fadd_rn(la[0], __fdiv_rn(__fmul_rn(-sc.x, m), denom));
        la[0] = p; la[1] = m; la[2] = v;
        *alpha = expf(p);
        *const_cast<int *>(round_idx) += 1;
    }
}

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_sacd {
    prl_sacd_cfg cfg;
    int Pa, Pc;
    int aW1, ab1, aW2, ab2, aW3, ab3;
    int cW1, cb1, cW2, cb2, cW3, cb3;
    float *actor, *actor_m, *actor_v, *actor_x;
    float *critic, *critic_m, *critic_v, *critic_x, *critic_t;
    float *log_alpha, *alpha;
    int64_t adam_step;
    // workspace
    float *S, *S2, *R, *T, *h1, *h2, *logits, *dlogit, *ent, *dh2, *dh1, *P, *c1, *c2, *q, *c1a, *c2a, *dq, *dc2, *dc1, *y, *qa, *g_actor, *g_critic;
    int *act, *cnt, *ids;
    int32_t *slots, *logical;
    float2 *scal_a, *scal_c, *scal_e;
    SacdCall *call;
    int *round_idx;
    bool use_graph;
    cudaGraphExec_t graph_exec;
    int graph_batch;
    const uint32_t *graph_buf;
    int launches_per_round;
    float2 *scal_host[2];
    cudaEvent_t scal_done[2];
    int scal_next;
    int64_t last_launches;
};

static int64_t al64(int64_t x) { return (x + 255) / 256 * 256; }

static void sacd_layout(prl_sacd *s) {
    const prl_sacd_cfg &c = s->cfg;
    int o = 0;
    s->aW1 = o; o += c.actor_h1 * c.obs_dim; s->ab1 = o; o += c.actor_h1;
    s->aW2 = o; o += c.actor_h2 * c.actor_h1; s->ab2 = o; o += c.actor_h2;
    s->aW3 = o; o += c.n_actions * c.actor_h2; s->ab3 = o; o += c.n_actions;
    s->Pa = o;
    const int D = c.obs_dim + c.n_actions;
    o = 0;
    s->cW1 = o; o += c.critic_h1 * D; s->cb1 = o; o += c.critic_h1;
    s->cW2 = o; o += c.critic_h2 * c.critic_h1; s->cb2 = o; o += c.critic_h2;
    s->cW3 = o; o += c.critic_h2; s->cb3 = o; o += 1;
    s->Pc = o;
}

static int sacd_check(const prl_sacd_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->actor_h1 > 0 && c->actor_h2 > 0 && c->critic_h1 > 0 && c->critic_h2 > 0, "dimensions must be positive");
    PRL_REQUIRE(c->n_actions > 0 && c->n_actions <= kMaxA, "n_actions must be in [1, 255]");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    return PRL_OK;
}

extern "C" int64_t prl_sacd_actor_param_count(const prl_sacd_cfg *c) {
    if (sacd_check(c)) return -1;
    prl_sacd t; t.cfg = *c; sacd_layout(&t);
    return t.Pa;
}
extern "C" int64_t prl_sacd_critic_param_count(const prl_sacd_cfg *c) {
    if (sacd_check(c)) return -1;
    prl_sacd t; t.cfg = *c; sacd_layout(&t);
    return t.Pc;
}

struct SacdWs { int64_t off[40]; int64_t total; };
static SacdWs sacd_ws(const prl_sacd_cfg *c, int Pa, int Pc) {
    SacdWs w; int64_t o = 0; int k = 0;
    const int64_t B = c->max_batch, A = c->n_actions, O = c->obs_dim, BA = B * A;
    auto add = [&](int64_t words) { w.off[k++] = o; o = al64(o + words * 4); };
    add(B * O); add(B * O); add(B); add(B);                                                      // S S2 R T
    add(B * c->actor_h1); add(B * c->actor_h2); add(BA); add(BA); add(B);                        // h1 h2 logits dlogit ent
    add(B * c->actor_h2); add(B * c->actor_h1);                                                  // dh2 dh1
    add(2 * B * c->critic_h1); add(2 * BA * c->critic_h1); add(2 * BA * c->critic_h2); add(2 * BA);   // P c1 c2 q
    add(2 * B * c->critic_h1); add(2 * B * c->critic_h2); add(2 * B);                           // c1a c2a dq
    add(2 * B * c->critic_h2); add(2 * B * c->critic_h1); add(B); add(2 * B);                    // dc2 dc1 y qa
    add(Pa); add(2 * (int64_t)Pc);                                                               // g_actor g_critic
    add(B); add(B); add(BA);                                                                     // act cnt ids (int32)
    add((int64_t)c->max_rounds * B); add((int64_t)c->max_rounds * B);                           // slots logical (int32)
    add(6 * (int64_t)c->max_rounds + 64);                                                        // scal_a | scal_c | scal_e | call | round_idx
    w.total = o;
    return w;
}
extern "C" int64_t prl_sacd_workspace_bytes(const prl_sacd_cfg *c) {
    if (sacd_check(c)) return -1;
    prl_sacd t; t.cfg = *c; sacd_layout(&t);
    return sacd_ws(c, t.Pa, t.Pc).total;
}

extern "C" int prl_sacd_create(prl_sacd **out, const prl_sacd_cfg *cfg, float *actor_w, float *actor_m, float *actor_v, float *actor_vmax,
                               float *critic_w, float *critic_m, float *critic_v, float *critic_vmax, float *critic_target_w,
                               float *log_alpha3, float *alpha1, int64_t adam_step, void *workspace) {
    PRL_REQUIRE(out && actor_w && actor_m && actor_v && actor_vmax && critic_w && critic_m && critic_v && critic_vmax && critic_target_w &&
                    log_alpha3 && alpha1 && workspace, "null argument");
    int rc = sacd_check(cfg);
    if (rc) return rc;
    prl_sacd *s = new (std::nothrow) prl_sacd();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    sacd_layout(s);
    s->actor = actor_w; s->actor_m = actor_m; s->actor_v = actor_v; s->actor_x = actor_vmax;
    s->critic = critic_w; s->critic_m = critic_m; s->critic_v = critic_v; s->critic_x = critic_vmax; s->critic_t = critic_target_w;
    s->log_alpha = log_alpha3; s->alpha = alpha1;
    s->adam_step = adam_step;
    SacdWs w = sacd_ws(cfg, s->Pa, s->Pc);
    char *b = (char *)workspace;
    float **f[] = {&s->S, &s->S2, &s->R, &s->T, &s->h1, &s->h2, &s->logits, &s->dlogit, &s->ent, &s->dh2, &s->dh1, &s->P, &s->c1, &s->c2,
                   &s->q, &s->c1a, &s->c2a, &s->dq, &s->dc2, &s->dc1, &s->y, &s->qa, &s->g_actor, &s->g_critic};
    int k = 0;
    for (auto p : f) *p = (float *)(b + w.off[k++]);
    s->act = (int *)(b + w.off[k++]); s->cnt = (int *)(b + w.off[k++]); s->ids = (int *)(b + w.off[k++]);
    s->slots = (int32_t *)(b + w.off[k++]); s->logical = (int32_t *)(b + w.off[k++]);
    s->scal_a = (float2 *)(b + w.off[k++]); s->scal_c = s->scal_a + cfg->max_rounds; s->scal_e = s->scal_c + cfg->max_rounds;
    s->call = (SacdCall *)(s->scal_e + cfg->max_rounds); s->round_idx = (int *)(s->call + 1);
    s->scal_next = 0; s->use_graph = true; s->graph_exec = nullptr; s->graph_batch = 0; s->graph_buf = nullptr; s->last_launches = 0;
    s->launches_per_round = 0;
    static_assert(sizeof(SacdCall) + 4 <= 64 * 4, "call block fits the reserved tail");
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
        return fail(PRL_ECUDA, "prl_sacd_create: %s", cudaGetErrorString(e));
    }
    *out = s;
    return PRL_OK;
}
extern "C" int prl_sacd_destroy(prl_sacd *s) {
    if (!s) return PRL_OK;
    for (int i = 0; i < 2; i++) { cudaEventSynchronize(s->scal_done[i]); cudaEventDestroy(s->scal_done[i]); cudaFreeHost(s->scal_host[i]); }
    if (s->graph_exec) cudaGraphExecDestroy(s->graph_exec);
    delete s;
    return PRL_OK;
}
extern "C" int64_t prl_sacd_adam_step(const prl_sacd *s) { return s ? s->adam_step : -1; }

extern "C" int prl_sacd_set_lr(prl_sacd *s, double actor_lr, double critic_lr) {
    PRL_REQUIRE(s, "null handle");
    PRL_REQUIRE(actor_lr >= 0.0 && critic_lr >= 0.0, "learning rates must be non-negative");
    s->cfg.actor_lr = actor_lr;
    s->cfg.critic_lr = critic_lr;
    return PRL_OK;
}

// one learner round, launched (or captured) on `st`; everything round- or call-dependent is read through s->call / s->round_idx
static int sacd_round(prl_sacd *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_sacd_cfg &c = s->cfg;
    const int O = c.obs_dim, A = c.n_actions, D = O + A, BA = B * A;
    const int H1 = c.actor_h1, H2 = c.actor_h2, C1 = c.critic_h1, C2 = c.critic_h2;
    const long long Pc = s->Pc;
    // the decay factors of these two are overridden by call->decay_a / decay_c (k_adamw's decay pointer)
    const AdamHp h = adam_hp(0.0, c.beta1, c.beta2, c.eps, c.weight_decay);
    GemmLauncher L; L.st = st;
    const float *aw = s->actor, *cw = s->critic, *ct = s->critic_t;
    const long long sP = (long long)B * C1, sC1 = (long long)BA * C1, sC2 = (long long)BA * C2;
    const long long sA1 = (long long)B * C1, sA2 = (long long)B * C2;
    const int eb = 256;
    int small = 0;
    auto actor_forward = [&](const float *X) {
        L.fwd(mat(X, O), B, aw + s->aW1, O, 0, aw + s->ab1, 0, H1, O, true, s->h1, H1, 0);
        L.fwd(mat(s->h1, H1), B, aw + s->aW2, H1, 0, aw + s->ab2, 0, H2, H1, true, s->h2, H2, 0);
        L.fwd(mat(s->h2, H2), B, aw + s->aW3, H2, 0, aw + s->ab3, 0, A, H2, false, s->logits, A, 0);
    };
    auto critic_all = [&](const float *net, const float *X, const int *ids) {   // q[z][b*A + k], both critics (blockIdx.z)
        L.fwd(mat(X, O), B, net + s->cW1, D, Pc, net + s->cb1, Pc, C1, O, false, s->P, C1, sP, 2);
        dim3 ge((unsigned)(((long long)BA * C1 + eb - 1) / eb), 1, 2);
        k_fold_expand<<<ge, eb, 0, st>>>(B, A, C1, s->P, net + s->cW1 + O, D, Pc, ids, s->c1);
        L.fwd(mat(s->c1, C1, sC1), BA, net + s->cW2, C1, Pc, net + s->cb2, Pc, C2, C1, true, s->c2, C2, sC2, 2);
        L.fwd(mat(s->c2, C2, sC2), BA, net + s->cW3, C2, Pc, net + s->cb3, Pc, 1, C2, false, s->q, 1, BA, 2);
        small++;
    };
    const int dynamic = (buf->desc.flags & PRL_BUF_DYNAMIC_ACTIONS) ? 1 : 0;
    k_sacd_gather<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf->records, buf->lay, O, A, dynamic, s->call, s->round_idx, B, s->S, s->S2, s->act,
                                                        s->R, s->T, s->cnt, s->ids);
    // ---------------- actor step (actor_critic_base.py:333-343, soft_actor_critic.py _actor_loss)
    actor_forward(s->S);
    critic_all(cw, s->S, nullptr);
    k_sacd_pick<<<dim3(B, 1, 2), 128, 0, st>>>(B, A, C1, C2, s->act, s->c1, s->c2, s->q, s->c1a, s->c2a, s->qa);
    k_sacd_actor<<<1, 256, 0, st>>>(B, A, s->logits, s->q, s->alpha, s->dlogit, s->ent, s->call, s->round_idx);
    {
        float *ga = s->g_actor;
        L.bwd_w(s->dlogit, A, 0, B, A, mat(s->h2, H2), H2, ga + s->aW3, H2, 0, ga + s->ab3, 0);
        L.bwd_x(s->dlogit, A, 0, B, A, aw + s->aW3, H2, 0, 0, H2, s->dh2, H2, 0, s->h2, H2, 0, false);
        L.bwd_w(s->dh2, H2, 0, B, H2, mat(s->h1, H1), H1, ga + s->aW2, H1, 0, ga + s->ab2, 0);
        L.bwd_x(s->dh2, H2, 0, B, H2, aw + s->aW2, H1, 0, 0, H1, s->dh1, H1, 0, s->h1, H1, 0, false);
        L.bwd_w(s->dh1, H1, 0, B, H1, mat(s->S, O), O, ga + s->aW1, O, 0, ga + s->ab1, 0);
        k_adamw<<<(s->Pa + eb - 1) / eb, eb, 0, st>>>(s->Pa, s->actor, s->actor_m, s->actor_v, s->actor_x, ga, h, s->scal_a, s->round_idx,
                                                    nullptr, 0.f, 0.f, &s->call->decay_a);
    }
    // ---------------- critic step with the UPDATED actor and the critic target (:345-349)
    actor_forward(s->S2);
    critic_all(ct, s->S2, s->ids);
    k_sacd_target<<<(B + 127) / 128, 128, 0, st>>>(B, A, s->logits, s->q, s->cnt, s->alpha, (float)c.gamma, s->T, s->R, s->y);
    k_sacd_critic_loss<<<1, 256, 0, st>>>(B, s->qa, s->y, s->dq, s->call, s->round_idx);
    {
        float *gc = s->g_critic;
        L.bwd_w(s->dq, 1, B, B, 1, mat(s->c2a, C2, sA2), C2, gc + s->cW3, C2, Pc, gc + s->cb3, Pc, 2);
        dim3 g2((B * C2 + eb - 1) / eb, 1, 2);
        k_head_bwd<<<g2, eb, 0, st>>>(B, C2, s->dq, cw + s->cW3, Pc, s->c2a, s->dc2);
        L.bwd_w(s->dc2, C2, sA2, B, C2, mat(s->c1a, C1, sA1), C1, gc + s->cW2, C1, Pc, gc + s->cb2, Pc, 2);
        L.bwd_x(s->dc2, C2, sA2, B, C2, cw + s->cW2, C1, Pc, 0, C1, s->dc1, C1, sA1, s->c1a, C1, sA1, false, 2);
        L.bwd_w(s->dc1, C1, sA1, B, C1, mat(s->S, O), O, gc + s->cW1, D, Pc, gc + s->cb1, Pc, 2);   // state columns + b1
        k_fold_w1a_grad<<<dim3((C1 * A + eb - 1) / eb, 1, 2), eb, 0, st>>>(B, A, C1, s->act, s->dc1, gc + s->cW1 + O, D, Pc);
        const int n2p = 2 * s->Pc;
        k_adamw<<<(n2p + eb - 1) / eb, eb, 0, st>>>(n2p, s->critic, s->critic_m, s->critic_v, s->critic_x, gc, h, s->scal_c, s->round_idx,
                                                  s->critic_t, (float)c.tau, (float)(1.0 - c.tau), &s->call->decay_c);
    }
    // ---------------- entropy coefficient (soft_actor_critic.py learn_batch); also advances the round counter
    k_sacd_alpha<<<1, 256, 0, st>>>(B, s->ent, (float)c.target_entropy, s->log_alpha, s->alpha, (float)(1.0 - c.beta1), (float)c.beta2,
                                    (float)(1.0 - c.beta2), (float)c.entropy_eps, s->scal_e, s->round_idx, s->call, c.autotune);
    small += 10;   // gather, pick, actor loss, 2 x adamw, target, critic loss, head bwd, w1a grad, alpha (+ the expands)
    s->launches_per_round = L.count + small;
    return PRL_OK;
}

extern "C" int prl_sacd_learn(prl_sacd *s, prl_buf *buf, int rounds, int batch, float *out_actor_loss, float *out_critic_loss,
                              float *out_entropy_loss, int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && out_actor_loss && out_critic_loss && out_entropy_loss, "null argument");
    const prl_sacd_cfg &c = s->cfg;
    PRL_REQUIRE(rounds > 0 && rounds <= c.max_rounds && batch > 0 && batch <= c.max_batch, "rounds / batch outside the configured maxima");
    PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.obs_dim == c.obs_dim && buf->desc.n_actions == c.n_actions,
                "discrete SAC needs a discrete-action buffer with matching obs_dim / n_actions");
    PRL_REQUIRE(buf->shard_world <= 1, "the buffer is one shard of a multi-GPU buffer: discrete SAC samples local buffers only");
    cudaStream_t st = (cudaStream_t)stream_;
    int rc = prl_buf_sample_indices(buf, rounds, batch, out_logical ? out_logical : s->logical, s->slots, stream_);
    if (rc) return rc;
    // per-call block: Adam scalars of every round (as torch evaluates them in double), decay factors, pointers
    const int sb = s->scal_next; s->scal_next ^= 1;
    PRL_CUDA(cudaEventSynchronize(s->scal_done[sb]));
    float2 *hs = s->scal_host[sb];
    const int MR = c.max_rounds;
    for (int r = 0; r < rounds; r++) {
        const double step = (double)(s->adam_step + r + 1);
        const double bc1 = 1.0 - pow(c.beta1, step), bc2 = 1.0 - pow(c.beta2, step);
        hs[r] = make_float2((float)(c.actor_lr / bc1), (float)sqrt(bc2));
        hs[MR + r] = make_float2((float)(c.critic_lr / bc1), (float)sqrt(bc2));
        hs[2 * MR + r] = make_float2((float)(c.entropy_lr / bc1), (float)sqrt(bc2));
    }
    SacdCall *hc = reinterpret_cast<SacdCall *>(hs + 3 * (size_t)MR);
    hc->slots = s->slots; hc->out_actor = out_actor_loss; hc->out_critic = out_critic_loss; hc->out_entropy = out_entropy_loss;
    hc->decay_a = (float)(1.0 - c.actor_lr * c.weight_decay);
    hc->decay_c = (float)(1.0 - c.critic_lr * c.weight_decay);
    int *hround = reinterpret_cast<int *>(hc + 1);
    *hround = 0;
    // scal_a | scal_c | scal_e | call | round_idx are contiguous on the device in the same order
    PRL_CUDA(cudaMemcpyAsync(s->scal_a, hs, 3 * (size_t)MR * 8 + sizeof(SacdCall) + 4, cudaMemcpyHostToDevice, st));
    PRL_CUDA(cudaEventRecord(s->scal_done[sb], st));

    if (s->use_graph) {
        if (!s->graph_exec || s->graph_batch != batch || s->graph_buf != buf->records) {
            if (s->graph_exec) { cudaGraphExecDestroy(s->graph_exec); s->graph_exec = nullptr; }
            cudaStream_t cs;
            PRL_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
            cudaGraph_t graph = nullptr;
            cudaError_t e = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
            if (e == cudaSuccess) {
                sacd_round(s, buf, batch, cs);
                e = cudaStreamEndCapture(cs, &graph);
            }
            if (e == cudaSuccess) e = cudaGraphInstantiate(&s->graph_exec, graph, 0);
            if (graph) cudaGraphDestroy(graph);
            cudaStreamDestroy(cs);
            if (e != cudaSuccess) { s->graph_exec = nullptr; return fail(PRL_ECUDA, "prl_sacd_learn: graph capture failed: %s", cudaGetErrorString(e)); }
            s->graph_batch = batch; s->graph_buf = buf->records;
        }
        for (int r = 0; r < rounds; r++) PRL_CUDA(cudaGraphLaunch(s->graph_exec, st));
    } else {
        for (int r = 0; r < rounds; r++) {
            rc = sacd_round(s, buf, batch, st);
            if (rc) return rc;
        }
    }
    PRL_CUDA(cudaGetLastError());
    s->adam_step += rounds;
    s->last_launches = (int64_t)s->launches_per_round * rounds;
    return PRL_OK;
}
extern "C" int prl_sacd_set_graph(prl_sacd *s, int enable) {
    PRL_REQUIRE(s, "null handle");
    s->use_graph = enable != 0;
    return PRL_OK;
}
extern "C" int64_t prl_sacd_last_launches(const prl_sacd *s) { return s ? s->last_launches : -1; }
