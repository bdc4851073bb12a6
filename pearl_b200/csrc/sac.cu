// sac.cu — continuous Soft Actor-Critic learner (ContinuousSoftActorCritic.learn_batch driven by
// PolicyLearner.learn), replacing
//   policy_learners/sequential_decision_making/actor_critic_base.py:309-366   (actor step, critic step, soft update)
//   policy_learners/sequential_decision_making/soft_actor_critic_continuous.py:131-231 (losses, entropy autotune)
//   neural_networks/sequential_decision_making/actor_networks.py:29-51,488-591 (GaussianActorNetwork.sample_action)
//   neural_networks/sequential_decision_making/twin_critic.py:75-91, q_value_networks.py:152-174
//   utils/functional_utils/learning/critic_utils.py:103-122,170-203, torch.optim.AdamW(amsgrad=True)
//
// Round-1 structure: the step is a fixed sequence of launches of ONE generic tiled fp32 contraction
// kernel (forward y = act(x W^T + b), backward-data dx = dy W (* relu mask), backward-weight
// dW = dy^T x with the bias gradient as an implicit ones column; the state||action concat and the twin
// critics are handled inside the kernel: two-source operands, blockIdx.z = critic) plus small
// elementwise kernels for the tanh-Gaussian policy, the losses and AdamW.  fp32, fixed summation
// order (deterministic).  The tensor-core path of the DQN learner is not applied here yet.
#include <math.h>
#include <stdarg.h>

#include <new>

#include "common.cuh"
#include "gemm.cuh"
#include "rounds.cuh"

using namespace prl;

namespace {

// per-call pointers the captured round reads through (the graph itself never changes between calls)
struct SacCall {
    const float *noise;      // [rounds][2][B][A]
    const int32_t *slots;    // [rounds][B]
    float *out_actor, *out_critic, *out_entropy;
};

// ------------------------------------------------------------------ elementwise pieces
// batch rows of one round from the replay ring
__global__ void k_sac_gather(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int act, const SacCall *__restrict__ call,
                             const int *__restrict__ round_idx, int B, float *__restrict__ S, float *__restrict__ A, float *__restrict__ R,
                             float *__restrict__ S2, float *__restrict__ T) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    const int32_t *slots = call->slots + (size_t)(*round_idx) * B;
    const uint32_t *r = records + (size_t)slots[w] * L.record_words;
    for (int p = lane; p < obs; p += 32) {
        S[(size_t)w * obs + p] = __uint_as_float(r[L.off_state + p]);
        S2[(size_t)w * obs + p] = __uint_as_float(r[L.off_next_state + p]);
    }
    for (int p = lane; p < act; p += 32) A[(size_t)w * act + p] = __uint_as_float(r[L.off_action + p]);
    if (lane == 0) { R[w] = __uint_as_float(r[L.off_reward]); T[w] = (r[L.off_flags] & 1u) ? 1.f : 0.f; }
}

// GaussianActorNetwork.sample_action (actor_networks.py:551-591) with the rsample noise given
__global__ void k_sac_sample(int B, int A, const float *__restrict__ mean, const float *__restrict__ z, const SacCall *__restrict__ call,
                             const int *__restrict__ round_idx, int which, const float *__restrict__ low, const float *__restrict__ high,
                             float *__restrict__ action, float *__restrict__ na_out, float *__restrict__ std_out, float *__restrict__ logp) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float *noise = call->noise + (size_t)(2 * (*round_idx) + which) * B * A;
    float lp = 0.f;
    for (int d = 0; d < A; d++) {
        const size_t o = (size_t)b * A + d;
        const float log_std = -5.f + 3.5f * (tanhf(z[o]) + 1.f);
        const float sd = expf(log_std), eps = noise[o];
        const float sample = mean[o] + sd * eps;
        const float na = tanhf(sample);
        const float lo = low[d], hi = high[d], bound = (hi - lo) * 0.5f;
        action[o] = (((hi - lo) * (na + 1.0f)) / 2.f) + lo;
        na_out[o] = na; std_out[o] = sd;
        const float diff = sample - mean[o];
        float t = -(diff * diff) / (2.f * sd * sd) - log_std - 0.91893853320467274178f;   // Normal.log_prob
        t -= logf(bound * (1.f - na * na) + 1e-6f);
        lp += t;
    }
    logp[b] = lp;
}

// actor loss = mean(alpha * logp - min(q1, q2)); routes -1/B to the smaller critic
__global__ void k_sac_actor_loss(int B, const float *__restrict__ q, const float *__restrict__ logp, const float *__restrict__ alpha,
                                 float *__restrict__ dq, const SacCall *__restrict__ call, const int *__restrict__ round_idx) {
    __shared__ float red[256];
    float s = 0.f;
    const float al = *alpha, ib = 1.f / (float)B;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float q1 = q[b], q2 = q[B + b];
        const bool first = q1 <= q2;
        s += al * logp[b] - (first ? q1 : q2);
        dq[b] = first ? -ib : 0.f;
        dq[B + b] = first ? 0.f : -ib;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) call->out_actor[*round_idx] = red[0] * ib;
}

// gradients of the actor loss w.r.t. the two heads (mean, pre-tanh log-std z)
__global__ void k_sac_head_grads(int B, int A, const float *__restrict__ da /* [2][B][A] from both critics */,
                                 const float *__restrict__ na, const float *__restrict__ sd, const SacCall *__restrict__ call,
                                 const int *__restrict__ round_idx, const float *__restrict__ z, const float *__restrict__ low,
                                 const float *__restrict__ high, const float *__restrict__ alpha, float *__restrict__ dmean,
                                 float *__restrict__ dz) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= B * A) return;
    const float *noise = call->noise + (size_t)(2 * (*round_idx)) * B * A;
    const int d = e % A;
    const float al_b = *alpha / (float)B;
    const float lo = low[d], hi = high[d], bound = (hi - lo) * 0.5f;
    const float n = na[e];
    const float dact = da[e] + da[(size_t)B * A + e];
    // d/dna: action scaling, and -log(bound (1 - na^2) + 1e-6) inside log-prob
    const float dna = dact * (hi - lo) * 0.5f + al_b * (2.f * bound * n) / (bound * (1.f - n * n) + 1e-6f);
    const float du = dna * (1.f - n * n);                      // through tanh
    dmean[e] = du;
    const float dlogstd = du * sd[e] * noise[e] - al_b;         // sample = mean + std*eps ; -log_std term of log-prob
    const float tz = tanhf(z[e]);
    dz[e] = dlogstd * 3.5f * (1.f - tz * tz);
}

// y = (min(q1t, q2t) - alpha * logp') * gamma * (1 - terminated) + reward;  dq_i = (q_i - y) / B ; critic loss
__global__ void k_sac_target(int B, const float *__restrict__ qt, const float *__restrict__ logp2, const float *__restrict__ alpha,
                             float gamma, const float *__restrict__ term, const float *__restrict__ rew, float *__restrict__ y) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const float nq = fminf(qt[b], qt[B + b]) - (*alpha) * logp2[b];
    y[b] = __fadd_rn(__fmul_rn(__fmul_rn(nq, gamma), 1.f - term[b]), rew[b]);
}
__global__ void k_sac_critic_loss(int B, const float *__restrict__ q, const float *__restrict__ y, float *__restrict__ dq,
                                  const SacCall *__restrict__ call, const int *__restrict__ round_idx) {
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

// entropy coefficient: loss = mean(-exp(log_alpha) * (logp + target_entropy)); AdamW on the scalar; alpha = exp(log_alpha)
__global__ void k_sac_alpha(int B, const float *__restrict__ logp, float target_entropy, float *__restrict__ log_alpha /* [4]: w m v vmax */,
                            float *__restrict__ alpha, AdamHp h, const float2 *__restrict__ scal, const int *__restrict__ round_idx,
                            const SacCall *__restrict__ call, int autotune) {
    __shared__ float red[256];
    if (!autotune) {                       // fixed entropy coefficient: only the round counter advances
        if (threadIdx.x == 0) *const_cast<int *>(round_idx) += 1;
        return;
    }
    float s = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) s += logp[b] + target_entropy;
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) {
        const float mean = red[0] / (float)B, ea = expf(log_alpha[0]);
        call->out_entropy[*round_idx] = -ea * mean;
        const float g = -ea * mean;                 // d/dlog_alpha
        const float2 sc = scal[*round_idx];
        float mm = log_alpha[1], vv = log_alpha[2], xx = log_alpha[3];
        const float p = adamw1(log_alpha[0], mm, vv, xx, g, h, sc.x, sc.y);
        log_alpha[0] = p; log_alpha[1] = mm; log_alpha[2] = vv; log_alpha[3] = xx;
        *alpha = expf(p);
        *const_cast<int *>(round_idx) += 1;
    }
}

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_sac : Rounds<prl_sac, SacCall> {
    static constexpr const char *kFn = "prl_sac";
    static constexpr int kScal = 2;   // actor, critic
    prl_sac_cfg cfg;
    int Pa, Pc;                       // actor parameters; parameters of ONE critic
    // actor layout offsets
    int aW1, ab1, aW2, ab2, aWmu, abmu, aWsd, absd;
    int cW1, cb1, cW2, cb2, cW3, cb3; // critic layout offsets (within one critic)
    float *actor, *actor_m, *actor_v, *actor_x;
    float *critic, *critic_m, *critic_v, *critic_x, *critic_t;
    float *log_alpha, *alpha;         // log_alpha[4] = value, m, v, vmax ; alpha scalar
    const float *low, *high;
    // workspace
    float *S, *A, *R, *S2, *T, *h1, *h2, *mean, *z, *act_s, *na, *sd, *logp, *logp2, *c1, *c2, *q, *qt, *dq, *dc2, *dc1, *da, *dmean, *dz,
        *dh2, *dh1, *y, *g_actor, *g_critic;
    double &lr(int k) { return k == 0 ? cfg.actor_lr : cfg.critic_lr; }
    int buffer_ok(const prl_buf *buf) const {
        PRL_REQUIRE((buf->desc.flags & PRL_BUF_CONTINUOUS) && buf->desc.obs_dim == cfg.obs_dim && buf->desc.act_dim == cfg.act_dim,
                    "SAC needs a continuous-action buffer with matching dimensions");
        return PRL_OK;
    }
    static int round(prl_sac *s, prl_buf *buf, int B, cudaStream_t st);
};

static void sac_layout(prl_sac *s) {
    const prl_sac_cfg &c = s->cfg;
    int o = 0;
    s->aW1 = o; o += c.actor_h1 * c.obs_dim; s->ab1 = o; o += c.actor_h1;
    s->aW2 = o; o += c.actor_h2 * c.actor_h1; s->ab2 = o; o += c.actor_h2;
    s->aWmu = o; o += c.act_dim * c.actor_h2; s->abmu = o; o += c.act_dim;
    s->aWsd = o; o += c.act_dim * c.actor_h2; s->absd = o; o += c.act_dim;
    s->Pa = o;
    const int D = c.obs_dim + c.act_dim;
    o = 0;
    s->cW1 = o; o += c.critic_h1 * D; s->cb1 = o; o += c.critic_h1;
    s->cW2 = o; o += c.critic_h2 * c.critic_h1; s->cb2 = o; o += c.critic_h2;
    s->cW3 = o; o += c.critic_h2; s->cb3 = o; o += 1;
    s->Pc = o;
}

static int sac_check(const prl_sac_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->act_dim > 0 && c->actor_h1 > 0 && c->actor_h2 > 0 && c->critic_h1 > 0 && c->critic_h2 > 0,
                "dimensions must be positive");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    return PRL_OK;
}

extern "C" int64_t prl_sac_actor_param_count(const prl_sac_cfg *c) {
    if (sac_check(c)) return -1;
    prl_sac t; t.cfg = *c; sac_layout(&t);
    return t.Pa;
}
extern "C" int64_t prl_sac_critic_param_count(const prl_sac_cfg *c) {   // ONE critic; the twin vector holds two
    if (sac_check(c)) return -1;
    prl_sac t; t.cfg = *c; sac_layout(&t);
    return t.Pc;
}

// the workspace, in order; base == null: only its size
static int64_t sac_carve(prl_sac *s, void *base) {
    const prl_sac_cfg &c = s->cfg;
    const int64_t B = c.max_batch, A = c.act_dim, O = c.obs_dim;
    Carve w{(char *)base};
    w(s->S, B * O); w(s->A, B * A); w(s->R, B); w(s->S2, B * O); w(s->T, B);
    w(s->h1, B * c.actor_h1); w(s->h2, B * c.actor_h2); w(s->mean, B * A); w(s->z, B * A);
    w(s->act_s, B * A); w(s->na, B * A); w(s->sd, B * A); w(s->logp, B); w(s->logp2, B);
    w(s->c1, 2 * B * c.critic_h1); w(s->c2, 2 * B * c.critic_h2); w(s->q, 2 * B); w(s->qt, 2 * B);
    w(s->dq, 2 * B); w(s->dc2, 2 * B * c.critic_h2); w(s->dc1, 2 * B * c.critic_h1); w(s->da, 2 * B * A);
    w(s->dmean, B * A); w(s->dz, B * A); w(s->dh2, B * c.actor_h2); w(s->dh1, B * c.actor_h1); w(s->y, B);
    w(s->g_actor, s->Pa); w(s->g_critic, 2 * (int64_t)s->Pc);
    s->carve_tail(w, c.max_rounds, B);
    return w.bytes;
}
extern "C" int64_t prl_sac_workspace_bytes(const prl_sac_cfg *c) {
    if (sac_check(c)) return -1;
    prl_sac t; t.cfg = *c; sac_layout(&t);
    return sac_carve(&t, nullptr);
}

extern "C" int prl_sac_create(prl_sac **out, const prl_sac_cfg *cfg, float *actor_w, float *actor_m, float *actor_v, float *actor_vmax,
                              float *critic_w, float *critic_m, float *critic_v, float *critic_vmax, float *critic_target_w,
                              float *log_alpha4, float *alpha1, const float *low_dev, const float *high_dev, int64_t adam_step,
                              void *workspace) {
    PRL_REQUIRE(out && actor_w && actor_m && actor_v && actor_vmax && critic_w && critic_m && critic_v && critic_vmax &&
                    critic_target_w && log_alpha4 && alpha1 && low_dev && high_dev && workspace, "null argument");
    int rc = sac_check(cfg);
    if (rc) return rc;
    prl_sac *s = new (std::nothrow) prl_sac();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    sac_layout(s);
    s->actor = actor_w; s->actor_m = actor_m; s->actor_v = actor_v; s->actor_x = actor_vmax;
    s->critic = critic_w; s->critic_m = critic_m; s->critic_v = critic_v; s->critic_x = critic_vmax; s->critic_t = critic_target_w;
    s->log_alpha = log_alpha4; s->alpha = alpha1; s->low = low_dev; s->high = high_dev;
    s->adam_step = adam_step;
    sac_carve(s, workspace);
    return prl_sac::open(s, out);
}
extern "C" int prl_sac_destroy(prl_sac *s) { return prl_sac::destroy(s); }
extern "C" int64_t prl_sac_adam_step(const prl_sac *s) { return prl_sac::adam_step_of(s); }
extern "C" int prl_sac_set_graph(prl_sac *s, int enable) { return prl_sac::set_graph(s, enable); }
extern "C" int64_t prl_sac_last_launches(const prl_sac *s) { return prl_sac::last_launches_of(s); }

// one learner round, launched (or captured) on `st`; everything round-dependent is read on the device through
// s->call / s->round_idx
int prl_sac::round(prl_sac *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_sac_cfg &c = s->cfg;
    const float2 *scal_a = s->scal, *scal_c = s->scal + c.max_rounds;
    const int O = c.obs_dim, A = c.act_dim, D = O + A;
    const int H1 = c.actor_h1, H2 = c.actor_h2, C1 = c.critic_h1, C2 = c.critic_h2;
    const long long Pc = s->Pc;
    AdamHp ha{(float)(1.0 - c.actor_lr * c.weight_decay), (float)(1.0 - c.beta1), (float)c.beta2, (float)(1.0 - c.beta2), (float)c.eps};
    AdamHp hc{(float)(1.0 - c.critic_lr * c.weight_decay), (float)(1.0 - c.beta1), (float)c.beta2, (float)(1.0 - c.beta2), (float)c.eps};
    GemmLauncher L; L.st = st;
    const float *aw = s->actor, *cw = s->critic, *ct = s->critic_t;
    const long long sC1 = (long long)B * C1, sC2 = (long long)B * C2;
    auto actor_forward = [&](const float *X) {
        L.fwd(mat(X, O), B, aw + s->aW1, O, 0, aw + s->ab1, 0, H1, O, true, s->h1, H1, 0);
        L.fwd(mat(s->h1, H1), B, aw + s->aW2, H1, 0, aw + s->ab2, 0, H2, H1, true, s->h2, H2, 0);
        L.fwd(mat(s->h2, H2), B, aw + s->aWmu, H2, 0, aw + s->abmu, 0, A, H2, false, s->mean, A, 0);
        L.fwd(mat(s->h2, H2), B, aw + s->aWsd, H2, 0, aw + s->absd, 0, A, H2, false, s->z, A, 0);
    };
    auto critic_forward = [&](const float *net, const float *X, const float *Act, float *qout) {   // both critics (blockIdx.z)
        L.fwd(mat2(X, O, O, Act, A), B, net + s->cW1, D, Pc, net + s->cb1, Pc, C1, D, true, s->c1, C1, sC1, 2);
        L.fwd(mat(s->c1, C1, sC1), B, net + s->cW2, C1, Pc, net + s->cb2, Pc, C2, C1, true, s->c2, C2, sC2, 2);
        L.fwd(mat(s->c2, C2, sC2), B, net + s->cW3, C2, Pc, net + s->cb3, Pc, 1, C2, false, qout, 1, B, 2);
    };
    const int eb = 256;
    int small = 0;
    k_sac_gather<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf->records, buf->lay, O, A, s->call, s->round_idx, B, s->S, s->A, s->R, s->S2, s->T);
    // ---------------- actor step (actor_critic_base.py:333-343)
    actor_forward(s->S);
    k_sac_sample<<<(B + 127) / 128, 128, 0, st>>>(B, A, s->mean, s->z, s->call, s->round_idx, 0, s->low, s->high, s->act_s, s->na, s->sd, s->logp);
    critic_forward(cw, s->S, s->act_s, s->q);
    k_sac_actor_loss<<<1, 256, 0, st>>>(B, s->q, s->logp, s->alpha, s->dq, s->call, s->round_idx);
    {   // dQ/d(action) through both critics
        dim3 g2((B * C2 + eb - 1) / eb, 1, 2);
        k_head_bwd<<<g2, eb, 0, st>>>(B, C2, s->dq, cw + s->cW3, Pc, s->c2, s->dc2);
        L.bwd_x(s->dc2, C2, sC2, B, C2, cw + s->cW2, C1, Pc, 0, C1, s->dc1, C1, sC1, s->c1, C1, sC1, false, 2);
        L.bwd_x(s->dc1, C1, sC1, B, C1, cw + s->cW1, D, Pc, O, A, s->da, A, (long long)B * A, nullptr, 0, 0, false, 2);
    }
    k_sac_head_grads<<<(B * A + eb - 1) / eb, eb, 0, st>>>(B, A, s->da, s->na, s->sd, s->call, s->round_idx, s->z, s->low, s->high, s->alpha,
                                                         s->dmean, s->dz);
    {   // actor backward
        float *ga = s->g_actor;
        L.bwd_w(s->dmean, A, 0, B, A, mat(s->h2, H2), H2, ga + s->aWmu, H2, 0, ga + s->abmu, 0);
        L.bwd_w(s->dz, A, 0, B, A, mat(s->h2, H2), H2, ga + s->aWsd, H2, 0, ga + s->absd, 0);
        L.bwd_x(s->dmean, A, 0, B, A, aw + s->aWmu, H2, 0, 0, H2, s->dh2, H2, 0, nullptr, 0, 0, false);
        L.bwd_x(s->dz, A, 0, B, A, aw + s->aWsd, H2, 0, 0, H2, s->dh2, H2, 0, s->h2, H2, 0, true);
        L.bwd_w(s->dh2, H2, 0, B, H2, mat(s->h1, H1), H1, ga + s->aW2, H1, 0, ga + s->ab2, 0);
        L.bwd_x(s->dh2, H2, 0, B, H2, aw + s->aW2, H1, 0, 0, H1, s->dh1, H1, 0, s->h1, H1, 0, false);
        L.bwd_w(s->dh1, H1, 0, B, H1, mat(s->S, O), O, ga + s->aW1, O, 0, ga + s->ab1, 0);
        k_adamw<<<(s->Pa + eb - 1) / eb, eb, 0, st>>>(s->Pa, s->actor, s->actor_m, s->actor_v, s->actor_x, ga, ha, scal_a, s->round_idx, nullptr, 0.f, 0.f);
    }
    // ---------------- critic step with the UPDATED actor (:345-349; soft_actor_critic_continuous.py:155-205)
    actor_forward(s->S2);
    k_sac_sample<<<(B + 127) / 128, 128, 0, st>>>(B, A, s->mean, s->z, s->call, s->round_idx, 1, s->low, s->high, s->act_s, s->na, s->sd, s->logp2);
    critic_forward(ct, s->S2, s->act_s, s->qt);
    k_sac_target<<<(B + eb - 1) / eb, eb, 0, st>>>(B, s->qt, s->logp2, s->alpha, (float)c.gamma, s->T, s->R, s->y);
    critic_forward(cw, s->S, s->A, s->q);
    k_sac_critic_loss<<<1, 256, 0, st>>>(B, s->q, s->y, s->dq, s->call, s->round_idx);
    {
        float *gc = s->g_critic;
        L.bwd_w(s->dq, 1, B, B, 1, mat(s->c2, C2, sC2), C2, gc + s->cW3, C2, Pc, gc + s->cb3, Pc, 2);
        dim3 g2((B * C2 + eb - 1) / eb, 1, 2);
        k_head_bwd<<<g2, eb, 0, st>>>(B, C2, s->dq, cw + s->cW3, Pc, s->c2, s->dc2);
        L.bwd_w(s->dc2, C2, sC2, B, C2, mat(s->c1, C1, sC1), C1, gc + s->cW2, C1, Pc, gc + s->cb2, Pc, 2);
        L.bwd_x(s->dc2, C2, sC2, B, C2, cw + s->cW2, C1, Pc, 0, C1, s->dc1, C1, sC1, s->c1, C1, sC1, false, 2);
        L.bwd_w(s->dc1, C1, sC1, B, C1, mat2(s->S, O, O, s->A, A), D, gc + s->cW1, D, Pc, gc + s->cb1, Pc, 2);
        const int n2p = 2 * s->Pc;
        k_adamw<<<(n2p + eb - 1) / eb, eb, 0, st>>>(n2p, s->critic, s->critic_m, s->critic_v, s->critic_x, gc, hc, scal_c, s->round_idx,
                                                  s->critic_t, (float)c.tau, (float)(1.0 - c.tau));
    }
    small = 12;
    // ---------------- entropy coefficient (soft_actor_critic_continuous.py:134-147); also advances the round counter
    k_sac_alpha<<<1, 256, 0, st>>>(B, s->logp, -(float)A, s->log_alpha, s->alpha, hc, scal_c, s->round_idx, s->call, c.autotune);
    s->launches_per_round = L.count + small;
    return PRL_OK;
}

extern "C" int prl_sac_learn(prl_sac *s, prl_buf *buf, int rounds, int batch, const float *noise_dev, float *out_actor_loss,
                             float *out_critic_loss, float *out_entropy_loss, int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && noise_dev && out_actor_loss && out_critic_loss && out_entropy_loss, "null argument");
    SacCall call{};
    call.noise = noise_dev; call.out_actor = out_actor_loss; call.out_critic = out_critic_loss; call.out_entropy = out_entropy_loss;
    return prl_sac::learn(s, buf, rounds, batch, 0, out_logical, call, stream_);
}
