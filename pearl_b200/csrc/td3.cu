// td3.cu — the deterministic actor-critic learners TD3 and DDPG (TD3.learn_batch / ActorCriticBase.learn_batch driven by
// PolicyLearner.learn), replacing
//   policy_learners/sequential_decision_making/td3.py:106-202         delayed actor + target updates, clipped target noise
//   policy_learners/sequential_decision_making/ddpg.py:105-157        actor loss -mean Q1(s, pi(s)), twin critic loss
//   policy_learners/sequential_decision_making/actor_critic_base.py:309-366  step order, soft target updates
//   neural_networks/sequential_decision_making/actor_networks.py:29-51,448-485  VanillaContinuousActorNetwork, action_scaling
//   neural_networks/sequential_decision_making/twin_critic.py:75-91, utils/functional_utils/learning/critic_utils.py:103-122,170-203
// DDPG is the same step with actor_update_freq = 1 and no target noise (this reference trains a twin critic for DDPG too).
// TD3BC (td3.py:241-318) is TD3 with a behaviour-cloning term in the actor loss: a handle made by prl_td3bc_create also runs
// the behaviour network on S and replaces the actor-loss kernel by k_td3bc_actor_loss.  learn_batch (buf == null) reads the
// caller's dense batch from the call block instead of gathering from the ring.
// Same launch structure as the SAC learner (sac.cu): one round = a fixed sequence of launches of the tiled contraction
// kernel (gemm.cuh) plus small elementwise kernels, everything round-dependent read on the device through a per-call
// block; the rounds with and without the actor update are captured as two CUDA graphs (rounds.cuh) and replayed.
#include <math.h>
#include <stdarg.h>

#include <new>

#include "common.cuh"
#include "gemm.cuh"
#include "rounds.cuh"

using namespace prl;

namespace {

struct Td3Call {
    const float *noise;      // [rounds][B][A] target-policy noise (torch.normal draws), or null (DDPG)
    const int32_t *slots;    // [rounds][B]
    float *out_actor, *out_critic;
    // learn_batch: the caller's dense batch
    const float *d_state, *d_action, *d_reward, *d_next_state;
    const uint8_t *d_term;
    float alpha_bc;          // TD3BC: read every call, never baked into a captured round
    int shape;               // 1: train on reward - fp32(lambda) * cost (prl_td3_set_cost_lambda); read every call
    double lambda;
};

// records == null: copy the caller's dense batch from the call block instead of gathering from the ring
// off_cost >= 0: the ring's cost word; with call->shape the reward is ActorCriticBase.preprocess_batch's
// reward - lambda * cost, two fp32 roundings as torch does them (a Python float times an fp32 tensor is an fp32 product)
__global__ void k_td3_gather(const uint32_t *__restrict__ records, prl_buf_layout L, int off_cost, int obs, int act, const Td3Call *__restrict__ call,
                             const int *__restrict__ round_idx, int B, float *__restrict__ S, float *__restrict__ A, float *__restrict__ R,
                             float *__restrict__ S2, float *__restrict__ T) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    if (!records) {
        for (int p = lane; p < obs; p += 32) {
            S[(size_t)w * obs + p] = call->d_state[(size_t)w * obs + p];
            S2[(size_t)w * obs + p] = call->d_next_state[(size_t)w * obs + p];
        }
        for (int p = lane; p < act; p += 32) A[(size_t)w * act + p] = call->d_action[(size_t)w * act + p];
        if (lane == 0) { R[w] = call->d_reward[w]; T[w] = call->d_term[w] ? 1.f : 0.f; }
        return;
    }
    const int32_t *slots = call->slots + (size_t)(*round_idx) * B;
    const uint32_t *r = records + (size_t)slots[w] * L.record_words;
    for (int p = lane; p < obs; p += 32) {
        S[(size_t)w * obs + p] = __uint_as_float(r[L.off_state + p]);
        S2[(size_t)w * obs + p] = __uint_as_float(r[L.off_next_state + p]);
    }
    for (int p = lane; p < act; p += 32) A[(size_t)w * act + p] = __uint_as_float(r[L.off_action + p]);
    if (lane == 0) {
        float rw = __uint_as_float(r[L.off_reward]);
        if (off_cost >= 0 && call->shape) rw = __fsub_rn(rw, __fmul_rn((float)call->lambda, __uint_as_float(r[off_cost])));
        R[w] = rw;
        T[w] = (r[L.off_flags] & 1u) ? 1.f : 0.f;
    }
}

// VanillaContinuousActorNetwork.sample_action: tanh head, action_scaling (actor_networks.py:29-51,475-485);
// target policy (td3.py:150-175): + clamp(noise, +-clip) * (high - low) / 2, clamped to the box
__global__ void k_td3_act(int B, int A, const float *__restrict__ pre, const float *__restrict__ low, const float *__restrict__ high,
                          const Td3Call *__restrict__ call, const int *__restrict__ round_idx, int with_noise, float clip,
                          float *__restrict__ action, float *__restrict__ na_out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= B * A) return;
    const int d = e % A;
    const float lo = low[d], hi = high[d];
    const float na = tanhf(pre[e]);
    float a = (((hi - lo) * (na + 1.0f)) / 2.f) + lo;
    if (with_noise && call->noise) {
        float nz = call->noise[(size_t)(*round_idx) * B * A + e];
        nz = fminf(fmaxf(nz, -clip), clip) * (hi - lo) / 2.f;
        a = fminf(fmaxf(a + nz, lo), hi);
    }
    action[e] = a;
    if (na_out) na_out[e] = na;
}

// actor loss = -mean(q1); dq1 = -1/B
__global__ void k_td3_actor_loss(int B, const float *__restrict__ q1, float *__restrict__ dq, const Td3Call *__restrict__ call,
                                 const int *__restrict__ round_idx, float *__restrict__ last_actor_loss) {
    __shared__ float red[256];
    float s = 0.f;
    const float ib = 1.f / (float)B;
    for (int b = threadIdx.x; b < B; b += blockDim.x) { s -= q1[b]; dq[b] = -ib; }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) { *last_actor_loss = red[0] * ib; call->out_actor[*round_idx] = red[0] * ib; }
}
// TD3BC actor loss (td3.py:298-318): b = behavior_policy(s) is VanillaContinuousActorNetwork.forward, the raw tanh output
// in [-1, 1] and NOT scaled to the box (actor_networks.py:472-473), while a = sample_action(s) is scaled;
// lambda = alpha_bc / mean|q1| (detached), loss = mean((a - b)^2) over B*A - lambda mean(q1).
// dq1 = -lambda / B; bc[e] = b (the head gradient adds 2 (a - b) / (B A)).  One CTA, fixed order.
__global__ void __launch_bounds__(256) k_td3bc_actor_loss(int B, int A, const float *__restrict__ q1, const float *__restrict__ a,
                                                         const float *__restrict__ bpre, float *__restrict__ bc, float *__restrict__ dq,
                                                         const Td3Call *__restrict__ call, const int *__restrict__ round_idx,
                                                         float *__restrict__ last_actor_loss) {
    __shared__ float red[3][256];
    __shared__ float lam;
    float sa = 0.f, sq = 0.f, sd = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) { sa += fabsf(q1[b]); sq += q1[b]; }
    for (int e = threadIdx.x; e < B * A; e += blockDim.x) {
        const float bb = tanhf(bpre[e]), d = a[e] - bb;
        bc[e] = bb;
        sd += d * d;
    }
    red[0][threadIdx.x] = sa; red[1][threadIdx.x] = sq; red[2][threadIdx.x] = sd;
    __syncthreads();
    for (int o = 128; o; o >>= 1) {
        if (threadIdx.x < o)
            for (int k = 0; k < 3; k++) red[k][threadIdx.x] += red[k][threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float l = call->alpha_bc / (red[0][0] / (float)B);
        const float loss = red[2][0] / (float)(B * A) - l * (red[1][0] / (float)B);
        lam = l;
        *last_actor_loss = loss;
        call->out_actor[*round_idx] = loss;
    }
    __syncthreads();
    const float g = -lam / (float)B;
    for (int b = threadIdx.x; b < B; b += blockDim.x) dq[b] = g;
}
// rounds without an actor update report the last actor loss again (td3.py:128)
__global__ void k_td3_repeat_actor_loss(const Td3Call *__restrict__ call, const int *__restrict__ round_idx, const float *__restrict__ last) {
    call->out_actor[*round_idx] = *last;
}
// d(pre) = d(action) * (high - low) / 2 * (1 - tanh^2); bc != null (TD3BC): d(action) += 2 (a - b) / (B A)
__global__ void k_td3_head_grad(int B, int A, const float *__restrict__ da, const float *__restrict__ na, const float *__restrict__ low,
                                const float *__restrict__ high, const float *__restrict__ act, const float *__restrict__ bc,
                                float *__restrict__ dpre) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= B * A) return;
    const int d = e % A;
    const float n = na[e];
    float g = da[e];
    if (bc) g += 2.f * (act[e] - bc[e]) / (float)(B * A);
    dpre[e] = g * ((high[d] - low[d]) * 0.5f) * (1.f - n * n);
}
// y = min(q1t, q2t) * gamma * (1 - terminated) + reward
__global__ void k_td3_target(int B, const float *__restrict__ qt, float gamma, const float *__restrict__ term, const float *__restrict__ rew,
                             float *__restrict__ y) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    y[b] = __fadd_rn(__fmul_rn(__fmul_rn(fminf(qt[b], qt[B + b]), gamma), 1.f - term[b]), rew[b]);
}
__global__ void k_td3_critic_loss(int B, const float *__restrict__ q, const float *__restrict__ y, float *__restrict__ dq,
                                  const Td3Call *__restrict__ call, const int *__restrict__ round_idx) {
    __shared__ float red[256];
    float s = 0.f;
    const float ib = 1.f / (float)B;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float e1 = q[b] - y[b], e2 = q[B + b] - y[b];
        s += e1 * e1 + e2 * e2;
        dq[b] = e1 * ib;            // d/dq1 of (mse1 + mse2) / 2
        dq[B + b] = e2 * ib;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) call->out_critic[*round_idx] = red[0] * ib * 0.5f;
}
__global__ void k_td3_soft_update(int n, float *__restrict__ target, const float *__restrict__ src, float tau, float omtau) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) target[i] = __fadd_rn(__fmul_rn(tau, src[i]), __fmul_rn(omtau, target[i]));
}
__global__ void k_td3_bump(int *round_idx, int *actor_round_idx, int actor_updated) {
    *round_idx += 1;
    if (actor_updated) *actor_round_idx += 1;
}

}  // namespace

struct prl_td3 : Rounds<prl_td3, Td3Call> {
    static constexpr const char *kFn = "prl_td3";
    // actor, critic; round_idx, actor_round_idx; {ring, dense batch} x {with, without the actor update}
    static constexpr int kScal = 2, kCounters = 2, kGraphs = 4;
    prl_td3_cfg cfg;
    prl_td3bc_cfg bc{};                // TD3BC: the behaviour network's hidden widths (0: TD3 / DDPG)
    const float *behavior = nullptr;   // TD3BC: flat W1 b1 W2 b2 W3 b3 of the behaviour network
    int Pa, Pc;                        // actor parameters; parameters of ONE critic
    int aW1, ab1, aW2, ab2, aW3, ab3;
    int cW1, cb1, cW2, cb2, cW3, cb3;
    float *actor, *actor_m, *actor_v, *actor_x, *actor_t;
    float *critic, *critic_m, *critic_v, *critic_x, *critic_t;
    const float *low, *high;
    int64_t actor_step;                // the actor optimizer's step count; adam_step counts the critic's
    float alpha_bc = 2.5f;             // TD3BC: copied into each call block
    int shape = 0;                     // prl_td3_set_cost_lambda: copied into the call blocks of prl_td3_learn
    double lambda = 0.0;
    float *S, *A, *R, *S2, *T, *h1, *h2, *pre, *act_s, *na, *c1, *c2, *q, *qt, *dq, *dc2, *dc1, *da, *dpre, *dh2, *dh1, *y, *g_actor,
        *g_critic, *last_actor_loss;
    float *bb1, *bb2, *bpre, *bact;    // TD3BC: the behaviour network's activations, pre-tanh output, tanh output
    bool is_bc() const { return behavior != nullptr; }
    int buffer_ok(const prl_buf *buf) const {
        PRL_REQUIRE((buf->desc.flags & PRL_BUF_CONTINUOUS) && buf->desc.obs_dim == cfg.obs_dim && buf->desc.act_dim == cfg.act_dim,
                    "TD3 / DDPG need a continuous-action buffer with matching dimensions");
        return PRL_OK;
    }
    // 1: round r updates the actor.  PolicyLearner.learn increments _training_steps before learn_batch
    // (policy_learner.py:183), TD3 tests `_training_steps % actor_update_freq == 0` (td3.py:121)
    int variant(int r) const { return cfg.actor_update_freq <= 1 || (steps0 + r) % cfg.actor_update_freq == 0 ? 1 : 0; }
    // the actor optimizer's own step count only advances on update rounds
    void fill_scal(float2 *hs, int rounds) {
        const prl_td3_cfg &c = cfg;
        int n_actor = 0;
        for (int r = 0; r < rounds; r++) {
            hs[c.max_rounds + r] = adam_scal(c.critic_lr, c.beta1, c.beta2, adam_step + r + 1);
            if (variant(r)) {
                hs[n_actor] = adam_scal(c.actor_lr, c.beta1, c.beta2, actor_step + n_actor + 1);
                n_actor++;
            }
        }
    }
    void fill_call(Td3Call &k) const { k.alpha_bc = alpha_bc; }
    int round_variant(prl_buf *buf, int B, int variant, cudaStream_t st);
};

static void td3_layout(prl_td3 *s) {
    const prl_td3_cfg &c = s->cfg;
    int o = 0;
    s->aW1 = o; o += c.actor_h1 * c.obs_dim; s->ab1 = o; o += c.actor_h1;
    s->aW2 = o; o += c.actor_h2 * c.actor_h1; s->ab2 = o; o += c.actor_h2;
    s->aW3 = o; o += c.act_dim * c.actor_h2; s->ab3 = o; o += c.act_dim;
    s->Pa = o;
    const int D = c.obs_dim + c.act_dim;
    o = 0;
    s->cW1 = o; o += c.critic_h1 * D; s->cb1 = o; o += c.critic_h1;
    s->cW2 = o; o += c.critic_h2 * c.critic_h1; s->cb2 = o; o += c.critic_h2;
    s->cW3 = o; o += c.critic_h2; s->cb3 = o; o += 1;
    s->Pc = o;
}
static int td3_check(const prl_td3_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->act_dim > 0 && c->actor_h1 > 0 && c->actor_h2 > 0 && c->critic_h1 > 0 && c->critic_h2 > 0,
                "dimensions must be positive");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0 && c->actor_update_freq >= 1, "max_batch / max_rounds / actor_update_freq must be positive");
    return PRL_OK;
}
extern "C" int64_t prl_td3_actor_param_count(const prl_td3_cfg *c) {
    if (td3_check(c)) return -1;
    prl_td3 t; t.cfg = *c; td3_layout(&t);
    return t.Pa;
}
extern "C" int64_t prl_td3_critic_param_count(const prl_td3_cfg *c) {   // ONE critic; the twin vector holds two
    if (td3_check(c)) return -1;
    prl_td3 t; t.cfg = *c; td3_layout(&t);
    return t.Pc;
}
// the workspace, in order; base == null: only its size
static int64_t td3_carve(prl_td3 *s, void *base) {
    const prl_td3_cfg &c = s->cfg;
    const int64_t B = c.max_batch, A = c.act_dim, O = c.obs_dim;
    Carve w{(char *)base};
    w(s->S, B * O); w(s->A, B * A); w(s->R, B); w(s->S2, B * O); w(s->T, B);
    w(s->h1, B * c.actor_h1); w(s->h2, B * c.actor_h2); w(s->pre, B * A); w(s->act_s, B * A); w(s->na, B * A);
    w(s->c1, 2 * B * c.critic_h1); w(s->c2, 2 * B * c.critic_h2); w(s->q, 2 * B); w(s->qt, 2 * B);
    w(s->dq, 2 * B); w(s->dc2, 2 * B * c.critic_h2); w(s->dc1, 2 * B * c.critic_h1); w(s->da, 2 * B * A);
    w(s->dpre, B * A); w(s->dh2, B * c.actor_h2); w(s->dh1, B * c.actor_h1); w(s->y, B);
    w(s->g_actor, s->Pa); w(s->g_critic, 2 * (int64_t)s->Pc); w(s->last_actor_loss, 4);
    const prl_td3bc_cfg &k = s->bc;
    w(s->bb1, B * k.behavior_h1); w(s->bb2, B * k.behavior_h2); w(s->bpre, k.behavior_h1 ? B * A : 0); w(s->bact, k.behavior_h1 ? B * A : 0);
    s->carve_tail(w, c.max_rounds, B);
    return w.bytes;
}
extern "C" int64_t prl_td3_workspace_bytes(const prl_td3_cfg *c) {
    if (td3_check(c)) return -1;
    prl_td3 t; t.cfg = *c; td3_layout(&t);
    return td3_carve(&t, nullptr);
}
static int td3bc_check(const prl_td3bc_cfg *bc) {
    PRL_REQUIRE(bc, "null TD3BC cfg");
    PRL_REQUIRE(bc->behavior_h1 > 0 && bc->behavior_h2 > 0, "the behaviour network's hidden widths must be positive");
    return PRL_OK;
}
extern "C" int64_t prl_td3bc_workspace_bytes(const prl_td3_cfg *c, const prl_td3bc_cfg *bc) {
    if (td3_check(c) || td3bc_check(bc)) return -1;
    prl_td3 t; t.cfg = *c; t.bc = *bc; td3_layout(&t);
    return td3_carve(&t, nullptr);
}

static int td3_open(prl_td3 **out, const prl_td3_cfg *cfg, const prl_td3bc_cfg *bc, const float *behavior_w, float *actor_w,
                    float *actor_m, float *actor_v, float *actor_vmax, float *actor_target_w, float *critic_w, float *critic_m,
                    float *critic_v, float *critic_vmax, float *critic_target_w, const float *low_dev, const float *high_dev,
                    int64_t actor_adam_step, int64_t critic_adam_step, void *workspace) {
    PRL_REQUIRE(out && actor_w && actor_m && actor_v && actor_vmax && actor_target_w && critic_w && critic_m && critic_v && critic_vmax &&
                    critic_target_w && low_dev && high_dev && workspace, "null argument");
    int rc = td3_check(cfg);
    if (rc) return rc;
    prl_td3 *s = new (std::nothrow) prl_td3();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    if (bc) { s->bc = *bc; s->behavior = behavior_w; }
    td3_layout(s);
    s->actor = actor_w; s->actor_m = actor_m; s->actor_v = actor_v; s->actor_x = actor_vmax; s->actor_t = actor_target_w;
    s->critic = critic_w; s->critic_m = critic_m; s->critic_v = critic_v; s->critic_x = critic_vmax; s->critic_t = critic_target_w;
    s->low = low_dev; s->high = high_dev;
    s->actor_step = actor_adam_step; s->adam_step = critic_adam_step;
    td3_carve(s, workspace);
    const cudaError_t e = cudaMemset(s->last_actor_loss, 0, 16);
    if (e != cudaSuccess) { delete s; return fail(PRL_ECUDA, "prl_td3_create: %s", cudaGetErrorString(e)); }
    return prl_td3::open(s, out);
}
extern "C" int prl_td3_create(prl_td3 **out, const prl_td3_cfg *cfg, float *actor_w, float *actor_m, float *actor_v, float *actor_vmax,
                              float *actor_target_w, float *critic_w, float *critic_m, float *critic_v, float *critic_vmax,
                              float *critic_target_w, const float *low_dev, const float *high_dev, int64_t actor_adam_step,
                              int64_t critic_adam_step, void *workspace) {
    return td3_open(out, cfg, nullptr, nullptr, actor_w, actor_m, actor_v, actor_vmax, actor_target_w, critic_w, critic_m, critic_v,
                    critic_vmax, critic_target_w, low_dev, high_dev, actor_adam_step, critic_adam_step, workspace);
}
extern "C" int prl_td3bc_create(prl_td3 **out, const prl_td3_cfg *cfg, const prl_td3bc_cfg *bc, const float *behavior_w, float *actor_w,
                                float *actor_m, float *actor_v, float *actor_vmax, float *actor_target_w, float *critic_w, float *critic_m,
                                float *critic_v, float *critic_vmax, float *critic_target_w, const float *low_dev, const float *high_dev,
                                int64_t actor_adam_step, int64_t critic_adam_step, void *workspace) {
    int rc = td3bc_check(bc);
    if (rc) return rc;
    PRL_REQUIRE(behavior_w, "null behaviour weights");
    return td3_open(out, cfg, bc, behavior_w, actor_w, actor_m, actor_v, actor_vmax, actor_target_w, critic_w, critic_m, critic_v,
                    critic_vmax, critic_target_w, low_dev, high_dev, actor_adam_step, critic_adam_step, workspace);
}
extern "C" int prl_td3_destroy(prl_td3 *s) { return prl_td3::destroy(s); }
extern "C" int64_t prl_td3_actor_adam_step(const prl_td3 *s) { return s ? s->actor_step : -1; }
extern "C" int64_t prl_td3_critic_adam_step(const prl_td3 *s) { return prl_td3::adam_step_of(s); }
extern "C" int prl_td3_set_graph(prl_td3 *s, int enable) { return prl_td3::set_graph(s, enable); }
extern "C" int64_t prl_td3_last_launches(const prl_td3 *s) { return prl_td3::last_launches_of(s); }
extern "C" int64_t prl_td3_graph_captures(const prl_td3 *s) { return s ? s->graphs.captures : -1; }
extern "C" int prl_td3_set_cost_lambda(prl_td3 *s, int enable, double lambda) {
    PRL_REQUIRE(s, "null handle");
    PRL_REQUIRE(!enable || isfinite(lambda), "lambda must be finite");
    s->shape = enable ? 1 : 0;
    s->lambda = enable ? lambda : 0.0;
    return PRL_OK;
}
extern "C" int prl_td3_set_alpha_bc(prl_td3 *s, double alpha_bc) {
    PRL_REQUIRE(s, "null handle");
    PRL_REQUIRE(s->is_bc(), "alpha_bc belongs to a TD3BC handle (prl_td3bc_create)");
    PRL_REQUIRE(isfinite(alpha_bc), "alpha_bc must be finite");
    s->alpha_bc = (float)alpha_bc;
    return PRL_OK;
}
// the actor loss that rounds without an actor update report (the reference's _last_actor_loss, td3.py:104,122)
extern "C" int prl_td3_set_last_actor_loss(prl_td3 *s, float value) {
    PRL_REQUIRE(s, "null handle");
    PRL_CUDA(cudaMemcpy(s->last_actor_loss, &value, sizeof(float), cudaMemcpyHostToDevice));
    return PRL_OK;
}

// one learner round, launched (or captured) on `st`; variant 1: with the actor update
int prl_td3::round_variant(prl_buf *buf, int B, int variant, cudaStream_t st) {
    prl_td3 *s = this;
    const bool update_actor = variant == 1;
    const prl_td3_cfg &c = s->cfg;
    const float2 *scal_a = s->scal, *scal_c = s->scal + c.max_rounds;
    int *actor_round_idx = s->round_idx + 1;
    const int O = c.obs_dim, A = c.act_dim, D = O + A;
    const int H1 = c.actor_h1, H2 = c.actor_h2, C1 = c.critic_h1, C2 = c.critic_h2;
    const long long Pc = s->Pc;
    AdamHp ha = adam_hp(c.actor_lr, c.beta1, c.beta2, c.eps, c.weight_decay), hc = adam_hp(c.critic_lr, c.beta1, c.beta2, c.eps, c.weight_decay);
    GemmLauncher L; L.st = st;
    const float *cw = s->critic, *ct = s->critic_t;
    const long long sC1 = (long long)B * C1, sC2 = (long long)B * C2;
    auto actor_forward = [&](const float *net, const float *X) {
        L.fwd(mat(X, O), B, net + s->aW1, O, 0, net + s->ab1, 0, H1, O, true, s->h1, H1, 0);
        L.fwd(mat(s->h1, H1), B, net + s->aW2, H1, 0, net + s->ab2, 0, H2, H1, true, s->h2, H2, 0);
        L.fwd(mat(s->h2, H2), B, net + s->aW3, H2, 0, net + s->ab3, 0, A, H2, false, s->pre, A, 0);
    };
    auto critic_forward = [&](const float *net, const float *X, const float *Act, float *qout, int nets) {
        L.fwd(mat2(X, O, O, Act, A), B, net + s->cW1, D, Pc, net + s->cb1, Pc, C1, D, true, s->c1, C1, sC1, nets);
        L.fwd(mat(s->c1, C1, sC1), B, net + s->cW2, C1, Pc, net + s->cb2, Pc, C2, C1, true, s->c2, C2, sC2, nets);
        L.fwd(mat(s->c2, C2, sC2), B, net + s->cW3, C2, Pc, net + s->cb3, Pc, 1, C2, false, qout, 1, B, nets);
    };
    const int eb = 256;
    int small = 0;
    // the cost word follows from the buffer's flags and layout, which the graph key compares
    int32_t off_cost = -1;
    if (buf && (buf->desc.flags & PRL_BUF_COST)) prl_buf_cost_offset(&buf->desc, &off_cost);
    k_td3_gather<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf ? buf->records : nullptr, buf ? buf->lay : prl_buf_layout{}, off_cost, O, A,
                                                        s->call, s->round_idx, B, s->S, s->A, s->R, s->S2, s->T);
    small++;
    if (update_actor) {
        // ---------------- actor step: maximise Q1(s, pi(s))   (ddpg.py:105-121)
        actor_forward(s->actor, s->S);
        k_td3_act<<<(B * A + eb - 1) / eb, eb, 0, st>>>(B, A, s->pre, s->low, s->high, s->call, s->round_idx, 0, 0.f, s->act_s, s->na);
        critic_forward(cw, s->S, s->act_s, s->q, 1);
        if (s->is_bc()) {
            // behavior_policy(s) under no_grad (td3.py:308-309), into its own scratch: h1 / h2 feed the actor's backward pass
            const int K1 = s->bc.behavior_h1, K2 = s->bc.behavior_h2;
            const float *bw = s->behavior;
            L.fwd(mat(s->S, O), B, bw, O, 0, bw + K1 * O, 0, K1, O, true, s->bb1, K1, 0);
            L.fwd(mat(s->bb1, K1), B, bw + K1 * O + K1, K1, 0, bw + K1 * O + K1 + K2 * K1, 0, K2, K1, true, s->bb2, K2, 0);
            L.fwd(mat(s->bb2, K2), B, bw + K1 * O + K1 + K2 * K1 + K2, K2, 0, bw + K1 * O + K1 + K2 * K1 + K2 + A * K2, 0, A, K2, false,
                  s->bpre, A, 0);
            k_td3bc_actor_loss<<<1, 256, 0, st>>>(B, A, s->q, s->act_s, s->bpre, s->bact, s->dq, s->call, s->round_idx, s->last_actor_loss);
        } else {
            k_td3_actor_loss<<<1, 256, 0, st>>>(B, s->q, s->dq, s->call, s->round_idx, s->last_actor_loss);
        }
        dim3 g1((B * C2 + eb - 1) / eb, 1, 1);
        k_head_bwd<<<g1, eb, 0, st>>>(B, C2, s->dq, cw + s->cW3, Pc, s->c2, s->dc2);
        L.bwd_x(s->dc2, C2, sC2, B, C2, cw + s->cW2, C1, Pc, 0, C1, s->dc1, C1, sC1, s->c1, C1, sC1, false, 1);
        L.bwd_x(s->dc1, C1, sC1, B, C1, cw + s->cW1, D, Pc, O, A, s->da, A, (long long)B * A, nullptr, 0, 0, false, 1);
        k_td3_head_grad<<<(B * A + eb - 1) / eb, eb, 0, st>>>(B, A, s->da, s->na, s->low, s->high, s->act_s, s->is_bc() ? s->bact : nullptr,
                                                              s->dpre);
        float *ga = s->g_actor;
        const float *aw = s->actor;
        L.bwd_w(s->dpre, A, 0, B, A, mat(s->h2, H2), H2, ga + s->aW3, H2, 0, ga + s->ab3, 0);
        L.bwd_x(s->dpre, A, 0, B, A, aw + s->aW3, H2, 0, 0, H2, s->dh2, H2, 0, s->h2, H2, 0, false);
        L.bwd_w(s->dh2, H2, 0, B, H2, mat(s->h1, H1), H1, ga + s->aW2, H1, 0, ga + s->ab2, 0);
        L.bwd_x(s->dh2, H2, 0, B, H2, aw + s->aW2, H1, 0, 0, H1, s->dh1, H1, 0, s->h1, H1, 0, false);
        L.bwd_w(s->dh1, H1, 0, B, H1, mat(s->S, O), O, ga + s->aW1, O, 0, ga + s->ab1, 0);
        k_adamw<<<(s->Pa + eb - 1) / eb, eb, 0, st>>>(s->Pa, s->actor, s->actor_m, s->actor_v, s->actor_x, ga, ha, scal_a, actor_round_idx,
                                                     nullptr, 0.f, 0.f);
        small += 5;
    } else {
        k_td3_repeat_actor_loss<<<1, 1, 0, st>>>(s->call, s->round_idx, s->last_actor_loss);
        small++;
    }
    // ---------------- critic step (td3.py:150-202 / ddpg.py:123-157): target action from the TARGET actor (+ clipped noise)
    actor_forward(s->actor_t, s->S2);
    k_td3_act<<<(B * A + eb - 1) / eb, eb, 0, st>>>(B, A, s->pre, s->low, s->high, s->call, s->round_idx, 1, (float)c.noise_clip, s->act_s, nullptr);
    critic_forward(ct, s->S2, s->act_s, s->qt, 2);
    k_td3_target<<<(B + eb - 1) / eb, eb, 0, st>>>(B, s->qt, (float)c.gamma, s->T, s->R, s->y);
    critic_forward(cw, s->S, s->A, s->q, 2);
    k_td3_critic_loss<<<1, 256, 0, st>>>(B, s->q, s->y, s->dq, s->call, s->round_idx);
    {
        float *gc = s->g_critic;
        L.bwd_w(s->dq, 1, B, B, 1, mat(s->c2, C2, sC2), C2, gc + s->cW3, C2, Pc, gc + s->cb3, Pc, 2);
        dim3 g2((B * C2 + eb - 1) / eb, 1, 2);
        k_head_bwd<<<g2, eb, 0, st>>>(B, C2, s->dq, cw + s->cW3, Pc, s->c2, s->dc2);
        L.bwd_w(s->dc2, C2, sC2, B, C2, mat(s->c1, C1, sC1), C1, gc + s->cW2, C1, Pc, gc + s->cb2, Pc, 2);
        L.bwd_x(s->dc2, C2, sC2, B, C2, cw + s->cW2, C1, Pc, 0, C1, s->dc1, C1, sC1, s->c1, C1, sC1, false, 2);
        L.bwd_w(s->dc1, C1, sC1, B, C1, mat2(s->S, O, O, s->A, A), D, gc + s->cW1, D, Pc, gc + s->cb1, Pc, 2);
        const int n2p = 2 * s->Pc;
        // the critic targets follow only on rounds with an actor update (td3.py:136-147); DDPG: every round
        k_adamw<<<(n2p + eb - 1) / eb, eb, 0, st>>>(n2p, s->critic, s->critic_m, s->critic_v, s->critic_x, gc, hc, scal_c, s->round_idx,
                                                  update_actor ? s->critic_t : nullptr, (float)c.critic_tau, (float)(1.0 - c.critic_tau));
    }
    small += 6;
    if (update_actor) {
        k_td3_soft_update<<<(s->Pa + eb - 1) / eb, eb, 0, st>>>(s->Pa, s->actor_t, s->actor, (float)c.actor_tau, (float)(1.0 - c.actor_tau));
        small++;
    }
    k_td3_bump<<<1, 1, 0, st>>>(s->round_idx, actor_round_idx, update_actor ? 1 : 0);
    small++;
    s->launches_per_round = L.count + small;
    return PRL_OK;
}

extern "C" int prl_td3_learn(prl_td3 *s, prl_buf *buf, int rounds, int batch, int64_t training_steps0, const float *noise_dev,
                             float *out_actor_loss, float *out_critic_loss, int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && out_actor_loss && out_critic_loss, "null argument");
    PRL_REQUIRE(!s->shape || (buf->desc.flags & PRL_BUF_COST),
                "cost-shaped rewards need a buffer with costs (PRL_BUF_COST): the reference fails on batch.cost = None");
    Td3Call call{};
    call.noise = noise_dev; call.out_actor = out_actor_loss; call.out_critic = out_critic_loss;
    call.shape = s->shape; call.lambda = s->lambda;
    const int rc = prl_td3::learn(s, buf, rounds, batch, training_steps0, out_logical, call, stream_);
    if (rc) return rc;
    for (int r = 0; r < rounds; r++) s->actor_step += s->variant(r);
    return PRL_OK;
}

// TD3.learn_batch / ActorCriticBase.learn_batch on the caller's dense batch: one round at `training_steps`, which the
// reference's learn_batch reads as it is (no increment, policy_learner.py:183 is in learn only)
extern "C" int prl_td3_learn_batch(prl_td3 *s, int batch, const float *state, const float *action, const float *reward,
                                   const float *next_state, const uint8_t *terminated, int64_t training_steps, const float *noise_dev,
                                   float *out_actor_loss, float *out_critic_loss, void *stream_) {
    PRL_REQUIRE(s && state && action && reward && next_state && terminated && out_actor_loss && out_critic_loss, "null argument");
    PRL_REQUIRE(training_steps >= 0, "training_steps must be non-negative");
    Td3Call call{};
    call.noise = noise_dev; call.out_actor = out_actor_loss; call.out_critic = out_critic_loss;
    call.d_state = state; call.d_action = action; call.d_reward = reward; call.d_next_state = next_state; call.d_term = terminated;
    const int rc = prl_td3::learn_batch(s, batch, training_steps, call, stream_);
    if (rc) return rc;
    s->actor_step += s->variant(0);
    return PRL_OK;
}
