// rc_safety.cu — the reward-constrained safety module's step (RCSafetyModuleCostCriticContinuousAction.learn, called by
// PearlAgent.learn after the policy learner's rounds), replacing
//   safety_modules/reward_constrained_safety_module.py:115-216   batch, cost-critic step, projected lambda step
//   utils/functional_utils/learning/critic_utils.py:103-122,170-203   twin Q values, twin MSE loss, soft target update
//   neural_networks/sequential_decision_making/actor_networks.py:29-51,475-485   sample_action of the (noise-free) actor
// One call = one sampled batch and one fixed launch sequence (captured as one CUDA graph, rounds.cuh):
//   gather S, A, cost, S', T | copy the policy's actor weights (their address travels in the per-call block, the
//   contractions take theirs from the workspace) | a' = actor(S') | y = min(Qc1', Qc2')(S', a') gamma_c (1 - T) + cost |
//   twin forward, loss, backward | k_adamw with the fused soft update of the target twin | a = actor(S) | the UPDATED twin
//   on (S, a) | one CTA: cq = mean(max(Qc1, Qc2)), then the float64 lambda step with its clamp.
// The twin layers and the backward chain are td3.cu's critic step; the kernels below are the few elementwise pieces.
#include <math.h>
#include <stdarg.h>

#include <new>

#include "common.cuh"
#include "gemm.cuh"
#include "rounds.cuh"

using namespace prl;

namespace {

struct RcCall {
    const int32_t *slots;     // [1][B]
    prl_rcsafety_step step;   // actor weights, box, lambda and its hyper-parameters, outputs
};

// one warp per row: S, A, cost, S', T of the sampled records
__global__ void k_rc_gather(const uint32_t *__restrict__ records, prl_buf_layout L, int off_cost, int obs, int act,
                            const RcCall *__restrict__ call, int B, float *__restrict__ S, float *__restrict__ A, float *__restrict__ C,
                            float *__restrict__ S2, float *__restrict__ T) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    const uint32_t *r = records + (size_t)call->slots[w] * L.record_words;
    for (int p = lane; p < obs; p += 32) {
        S[(size_t)w * obs + p] = __uint_as_float(r[L.off_state + p]);
        S2[(size_t)w * obs + p] = __uint_as_float(r[L.off_next_state + p]);
    }
    for (int p = lane; p < act; p += 32) A[(size_t)w * act + p] = __uint_as_float(r[L.off_action + p]);
    if (lane == 0) { C[w] = __uint_as_float(r[off_cost]); T[w] = (r[L.off_flags] & 1u) ? 1.f : 0.f; }
}

// the policy's actor weights, from the address of this call
__global__ void k_rc_load_actor(int n, const RcCall *__restrict__ call, float *__restrict__ dst) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = call->step.actor_w[i];
}

// VanillaContinuousActorNetwork.sample_action: tanh head scaled to the box, no noise (actor_networks.py:29-51,475-485)
__global__ void k_rc_act(int B, int A, const float *__restrict__ pre, const RcCall *__restrict__ call, float *__restrict__ action) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= B * A) return;
    const int d = e % A;
    const float lo = call->step.low[d], hi = call->step.high[d];
    action[e] = (((hi - lo) * (tanhf(pre[e]) + 1.0f)) / 2.f) + lo;
}

// y = min(q1t, q2t) * gamma_c * (1 - terminated) + cost   (reward_constrained_safety_module.py:183-192)
__global__ void k_rc_target(int B, const float *__restrict__ qt, float gamma, const float *__restrict__ term, const float *__restrict__ cost,
                            float *__restrict__ y) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    y[b] = __fadd_rn(__fmul_rn(__fmul_rn(fminf(qt[b], qt[B + b]), gamma), 1.f - term[b]), cost[b]);
}

// twin loss (mse1 + mse2) / 2 and its gradient dq = (q - y) / B; one CTA, fixed order; loss -> step.out[1]
__global__ void __launch_bounds__(256) k_rc_critic_loss(int B, const float *__restrict__ q, const float *__restrict__ y, float *__restrict__ dq,
                                                        const RcCall *__restrict__ call) {
    __shared__ float red[256];
    float s = 0.f;
    const float ib = 1.f / (float)B;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float e1 = q[b] - y[b], e2 = q[B + b] - y[b];
        s += e1 * e1 + e2 * e2;
        dq[b] = e1 * ib;
        dq[B + b] = e2 * ib;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) call->step.out[1] = (double)(red[0] * ib * 0.5f);
}

// cq = mean(max(q1, q2)) in fp32 (read back with .item()), then constraint_lambda_update (:130-160) in float64 with
// Python's evaluation order and max / min semantics; one CTA, fixed order
__global__ void __launch_bounds__(256) k_rc_lambda(int B, const float *__restrict__ q, double cost_gamma, const RcCall *__restrict__ call) {
    __shared__ float red[256];
    float s = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) s += fmaxf(q[b], q[B + b]);
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) {
        const prl_rcsafety_step &k = call->step;
        const double cq = (double)(red[0] / (float)B);
        double l = __dadd_rn(k.lambda_in, __dmul_rn(k.lr_lambda, __dsub_rn(__dmul_rn(cq, __dsub_rn(1.0, cost_gamma)), k.constraint_value)));
        l = 0.0 > l ? 0.0 : l;                    // max(l, 0.0)
        l = k.lambda_ub < l ? k.lambda_ub : l;    // min(l, ub)
        k.out[0] = l;
        k.out[2] = cq;
    }
}

}  // namespace

struct prl_rcsafety : Rounds<prl_rcsafety, RcCall> {
    static constexpr const char *kFn = "prl_rcsafety";
    struct Cfg : prl_rcsafety_cfg {
        int32_t max_rounds = 1;    // one sample per call
    } cfg;
    int Pa, Pc;                    // actor parameters; parameters of ONE cost critic
    int cW1, cb1, cW2, cb2, cW3, cb3;
    float *critic, *critic_m, *critic_v, *critic_x, *critic_t;
    float *S, *A, *Cst, *S2, *T, *actor, *h1, *h2, *pre, *act_s, *c1, *c2, *q, *qt, *dq, *dc2, *dc1, *y, *g_critic;
    double &lr(int) { return cfg.critic_lr; }
    int buffer_ok(const prl_buf *buf) const {
        PRL_REQUIRE((buf->desc.flags & PRL_BUF_CONTINUOUS) && buf->desc.obs_dim == cfg.obs_dim && buf->desc.act_dim == cfg.act_dim,
                    "the cost critic needs a continuous-action buffer with obs_dim = %d and act_dim = %d", cfg.obs_dim, cfg.act_dim);
        PRL_REQUIRE(buf->desc.flags & PRL_BUF_COST, "the cost critic needs a buffer with costs (PRL_BUF_COST)");
        PRL_REQUIRE(buf->shard_world <= 1, "the buffer is one shard of a multi-GPU buffer: the cost critic samples local buffers only");
        return PRL_OK;
    }
    static int round(prl_rcsafety *s, prl_buf *buf, int B, cudaStream_t st);
};

static void rc_layout(prl_rcsafety *s) {
    const prl_rcsafety_cfg &c = s->cfg;
    s->Pa = c.actor_h1 * c.obs_dim + c.actor_h1 + c.actor_h2 * c.actor_h1 + c.actor_h2 + c.act_dim * c.actor_h2 + c.act_dim;
    const int D = c.obs_dim + c.act_dim;
    int o = 0;
    s->cW1 = o; o += c.critic_h1 * D; s->cb1 = o; o += c.critic_h1;
    s->cW2 = o; o += c.critic_h2 * c.critic_h1; s->cb2 = o; o += c.critic_h2;
    s->cW3 = o; o += c.critic_h2; s->cb3 = o; o += 1;
    s->Pc = o;
}
static int rc_check(const prl_rcsafety_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->act_dim > 0 && c->actor_h1 > 0 && c->actor_h2 > 0 && c->critic_h1 > 0 && c->critic_h2 > 0,
                "dimensions must be positive");
    PRL_REQUIRE(c->max_batch > 0, "max_batch must be positive");
    PRL_REQUIRE(c->critic_lr >= 0.0, "the learning rate must be non-negative");
    return PRL_OK;
}
static int64_t rc_carve(prl_rcsafety *s, void *base) {
    const prl_rcsafety_cfg &c = s->cfg;
    const int64_t B = c.max_batch, A = c.act_dim, O = c.obs_dim;
    Carve w{(char *)base};
    w(s->S, B * O); w(s->A, B * A); w(s->Cst, B); w(s->S2, B * O); w(s->T, B); w(s->actor, s->Pa);
    w(s->h1, B * c.actor_h1); w(s->h2, B * c.actor_h2); w(s->pre, B * A); w(s->act_s, B * A);
    w(s->c1, 2 * B * c.critic_h1); w(s->c2, 2 * B * c.critic_h2); w(s->q, 2 * B); w(s->qt, 2 * B);
    w(s->dq, 2 * B); w(s->dc2, 2 * B * c.critic_h2); w(s->dc1, 2 * B * c.critic_h1); w(s->y, B); w(s->g_critic, 2 * (int64_t)s->Pc);
    s->carve_tail(w, s->cfg.max_rounds, B);
    return w.bytes;
}
extern "C" int64_t prl_rcsafety_param_count(const prl_rcsafety_cfg *c) {
    if (rc_check(c)) return -1;
    prl_rcsafety t; static_cast<prl_rcsafety_cfg &>(t.cfg) = *c; rc_layout(&t);
    return t.Pc;
}
extern "C" int64_t prl_rcsafety_workspace_bytes(const prl_rcsafety_cfg *c) {
    if (rc_check(c)) return -1;
    prl_rcsafety t; static_cast<prl_rcsafety_cfg &>(t.cfg) = *c; rc_layout(&t);
    return rc_carve(&t, nullptr);
}
extern "C" int prl_rcsafety_create(prl_rcsafety **out, const prl_rcsafety_cfg *cfg, float *critic_w, float *critic_m, float *critic_v,
                                   float *critic_vmax, float *critic_target_w, int64_t adam_step, void *workspace) {
    PRL_REQUIRE(out && critic_w && critic_m && critic_v && critic_vmax && critic_target_w && workspace, "null argument");
    PRL_REQUIRE(adam_step >= 0, "the AdamW step count must be non-negative");
    int rc = rc_check(cfg);
    if (rc) return rc;
    prl_rcsafety *s = new (std::nothrow) prl_rcsafety();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    static_cast<prl_rcsafety_cfg &>(s->cfg) = *cfg;
    rc_layout(s);
    s->critic = critic_w; s->critic_m = critic_m; s->critic_v = critic_v; s->critic_x = critic_vmax; s->critic_t = critic_target_w;
    s->adam_step = adam_step;
    rc_carve(s, workspace);
    return prl_rcsafety::open(s, out);
}
extern "C" int prl_rcsafety_destroy(prl_rcsafety *s) { return prl_rcsafety::destroy(s); }
extern "C" int64_t prl_rcsafety_adam_step(const prl_rcsafety *s) { return prl_rcsafety::adam_step_of(s); }
extern "C" int prl_rcsafety_set_graph(prl_rcsafety *s, int enable) { return prl_rcsafety::set_graph(s, enable); }
extern "C" int64_t prl_rcsafety_graph_captures(const prl_rcsafety *s) { return s ? s->graphs.captures : -1; }
extern "C" int64_t prl_rcsafety_last_launches(const prl_rcsafety *s) { return prl_rcsafety::last_launches_of(s); }

int prl_rcsafety::round(prl_rcsafety *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_rcsafety_cfg &c = s->cfg;
    const int O = c.obs_dim, A = c.act_dim, D = O + A;
    const int H1 = c.actor_h1, H2 = c.actor_h2, C1 = c.critic_h1, C2 = c.critic_h2;
    const long long Pc = s->Pc;
    const AdamHp hc = adam_hp(c.critic_lr, c.beta1, c.beta2, c.eps, c.weight_decay);
    GemmLauncher L; L.st = st;
    const float *cw = s->critic, *ct = s->critic_t, *aw = s->actor;
    const long long sC1 = (long long)B * C1, sC2 = (long long)B * C2;
    // the actor's flat layout: W1[H1][O] b1 W2[H2][H1] b2 W3[A][H2] b3
    const int aW2 = H1 * O + H1, aW3 = aW2 + H2 * H1 + H2;
    auto actor_act = [&](const float *X) {
        L.fwd(mat(X, O), B, aw, O, 0, aw + H1 * O, 0, H1, O, true, s->h1, H1, 0);
        L.fwd(mat(s->h1, H1), B, aw + aW2, H1, 0, aw + aW2 + H2 * H1, 0, H2, H1, true, s->h2, H2, 0);
        L.fwd(mat(s->h2, H2), B, aw + aW3, H2, 0, aw + aW3 + A * H2, 0, A, H2, false, s->pre, A, 0);
        k_rc_act<<<(B * A + 255) / 256, 256, 0, st>>>(B, A, s->pre, s->call, s->act_s);
    };
    auto critic_forward = [&](const float *net, const float *X, const float *Act, float *qout) {
        L.fwd(mat2(X, O, O, Act, A), B, net + s->cW1, D, Pc, net + s->cb1, Pc, C1, D, true, s->c1, C1, sC1, 2);
        L.fwd(mat(s->c1, C1, sC1), B, net + s->cW2, C1, Pc, net + s->cb2, Pc, C2, C1, true, s->c2, C2, sC2, 2);
        L.fwd(mat(s->c2, C2, sC2), B, net + s->cW3, C2, Pc, net + s->cb3, Pc, 1, C2, false, qout, 1, B, 2);
    };
    const int eb = 256;
    int32_t off_cost = -1;
    prl_buf_cost_offset(&buf->desc, &off_cost);     // buffer_ok checked PRL_BUF_COST; the graph key holds flags and layout
    k_rc_gather<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf->records, buf->lay, off_cost, O, A, s->call, B, s->S, s->A, s->Cst, s->S2, s->T);
    k_rc_load_actor<<<(s->Pa + eb - 1) / eb < 132 ? (s->Pa + eb - 1) / eb : 132, eb, 0, st>>>(s->Pa, s->call, s->actor);
    // ---------------- cost-critic step (:162-216): a' from the ONLINE actor, target from the target twin
    actor_act(s->S2);
    critic_forward(ct, s->S2, s->act_s, s->qt);
    k_rc_target<<<(B + eb - 1) / eb, eb, 0, st>>>(B, s->qt, (float)c.cost_gamma, s->T, s->Cst, s->y);
    critic_forward(cw, s->S, s->A, s->q);
    k_rc_critic_loss<<<1, 256, 0, st>>>(B, s->q, s->y, s->dq, s->call);
    float *gc = s->g_critic;
    L.bwd_w(s->dq, 1, B, B, 1, mat(s->c2, C2, sC2), C2, gc + s->cW3, C2, Pc, gc + s->cb3, Pc, 2);
    k_head_bwd<<<dim3((B * C2 + eb - 1) / eb, 1, 2), eb, 0, st>>>(B, C2, s->dq, cw + s->cW3, Pc, s->c2, s->dc2);
    L.bwd_w(s->dc2, C2, sC2, B, C2, mat(s->c1, C1, sC1), C1, gc + s->cW2, C1, Pc, gc + s->cb2, Pc, 2);
    L.bwd_x(s->dc2, C2, sC2, B, C2, cw + s->cW2, C1, Pc, 0, C1, s->dc1, C1, sC1, s->c1, C1, sC1, false, 2);
    L.bwd_w(s->dc1, C1, sC1, B, C1, mat2(s->S, O, O, s->A, A), D, gc + s->cW1, D, Pc, gc + s->cb1, Pc, 2);
    const int n2p = 2 * s->Pc;
    k_adamw<<<(n2p + eb - 1) / eb, eb, 0, st>>>(n2p, s->critic, s->critic_m, s->critic_v, s->critic_x, gc, hc, s->scal, s->round_idx,
                                              s->critic_t, (float)c.tau, (float)(1.0 - c.tau));
    // ---------------- lambda step (:130-160): the UPDATED twin at (S, actor(S))
    actor_act(s->S);
    critic_forward(cw, s->S, s->act_s, s->q);
    k_rc_lambda<<<1, 256, 0, st>>>(B, s->q, c.cost_gamma, s->call);
    s->launches_per_round = L.count + 9;
    return PRL_OK;
}

extern "C" int prl_rcsafety_learn(prl_rcsafety *s, prl_buf *buf, int batch, const prl_rcsafety_step *step, int32_t *out_logical,
                                  void *stream_) {
    PRL_REQUIRE(s && buf && step, "null argument");
    PRL_REQUIRE(step->actor_w && step->low && step->high && step->out, "null pointer in the step block");
    PRL_REQUIRE(isfinite(step->lambda_in) && isfinite(step->lr_lambda) && isfinite(step->constraint_value) && !isnan(step->lambda_ub),
                "lambda, lr_lambda, constraint_value and the upper bound must be numbers");
    RcCall call{};
    call.step = *step;
    return prl_rcsafety::learn(s, buf, 1, batch, 0, out_logical, call, stream_);
}
