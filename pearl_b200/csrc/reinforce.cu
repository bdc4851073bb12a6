// reinforce.cu — REINFORCE learner with a state-value baseline (REINFORCE.learn driven by PolicyLearner.learn), replacing
//   policy_learners/sequential_decision_making/reinforce.py:179-208   learn(): the return pass over the stored transitions
//   policy_learners/sequential_decision_making/reinforce.py:146-167   _actor_loss, _critic_loss
//   policy_learners/sequential_decision_making/actor_critic_base.py:309-366   learn_batch (actor step, then critic step)
//   neural_networks/sequential_decision_making/actor_networks.py:155-176     get_action_prob (softmax over ALL actions)
//   utils/functional_utils/learning/critic_utils.py:139-167                 single_critic_state_value_loss
//
// Return pass (prl_reinforce_returns): the critic at the newest transition's next_state, times (1 - terminated), then every
// stored reward added newest -> oldest in fp32.  The reference stores ONE tensor in every transition (an in-place += whose
// result each transition references), so every transition's return is that final sum R; there is no discount and no reset
// at episode ends.  The fold keeps the reference's operation order: given the same bootstrap, R is bit-identical.
//
// Round (captured once per (batch, buffer) into a CUDA graph and replayed): gather -> critic forward -> actor forward ->
// k_rf_loss -> actor backward + AdamW -> critic backward + AdamW -> round counter.  The actor loss of the reference is
// sum(nlp * (cum_reward - v)) with nlp of shape (B,) and cum_reward of shape (B, 1): a B x B broadcast, so the loss is
// sum_i sum_j nlp_j (R - v_j) = B sum_j nlp_j (R - v_j) and row j's gradient carries B (R - v_j).  The critic does not
// change between the two steps, so one critic forward serves both.  The AdamW step sizes and decay factors and the return
// pointer travel in the per-call block: prl_reinforce_set_lr needs no new capture.  fp32, fixed summation order, no float
// atomics: bit-reproducible run to run.
#include <math.h>
#include <stdarg.h>

#include <new>

#include "ac_nets.cuh"
#include "common.cuh"
#include "host_runtime.cuh"

using namespace prl;

namespace {

constexpr int kMaxA = 255;
constexpr int kFoldTile = 2048;   // rewards staged per shared-memory tile of the return fold

// per-call block the captured round reads through
struct RfCall {
    const int32_t *slots;        // [rounds][B]
    const float *ret;            // device f32: R (prl_reinforce_returns' first output)
    float *out_actor, *out_critic;
    float decay_a, decay_c;      // AdamW decoupled decay 1 - lr * weight_decay (actor, critic)
};

// The return fold, one CTA: cum = boot * (1 - terminated(newest)); cum += reward[i] for i = n-1 .. 0 (logical order, 0 =
// oldest).  Warps 1.. stage the next tile of rewards (one strided load per record, all in flight together) while lane 0
// of warp 0 adds the current tile in order.  out[0] = R, out[1] = the bootstrap term.
__global__ void __launch_bounds__(256) k_rf_fold(const uint32_t *__restrict__ records, prl_buf_layout L, int64_t head, int64_t cap, int64_t n,
                                                 const float *__restrict__ boot_value, float *__restrict__ out) {
    __shared__ __align__(16) float tile[2][kFoldTile];
    const int tid = threadIdx.x;
    const int64_t tiles = (n + kFoldTile - 1) / kFoldTile;
    // tile t holds logical indices n-1-t*kFoldTile .. down to max(0, n-(t+1)*kFoldTile), newest first
    auto stage = [&](int64_t t, int first, int step) {
        const int64_t top = n - 1 - t * kFoldTile;
        for (int k = first; k < kFoldTile; k += step) {
            const int64_t i = top - k;
            if (i >= 0) tile[t & 1][k] = __uint_as_float(records[(size_t)((head + i) % cap) * L.record_words + L.off_reward]);
        }
    };
    stage(0, tid, blockDim.x);
    __syncthreads();
    float cum = 0.f;
    if (tid == 0) {
        const uint32_t f = records[(size_t)((head + n - 1) % cap) * L.record_words + L.off_flags];
        cum = __fmul_rn(*boot_value, (f & 1u) ? 0.f : 1.f);   // critic(s').detach() * (~terminated)
        out[1] = cum;
    }
    for (int64_t t = 0; t < tiles; t++) {
        if (tid >= 32) {
            if (t + 1 < tiles) stage(t + 1, tid - 32, blockDim.x - 32);
        } else if (tid == 0) {
            const float *x = tile[t & 1];
            const int m = (int)(n - t * kFoldTile < kFoldTile ? n - t * kFoldTile : kFoldTile);
            int k = 0;
            for (; k + 8 <= m; k += 8) {
                const float4 a = *reinterpret_cast<const float4 *>(x + k), b = *reinterpret_cast<const float4 *>(x + k + 4);
                cum = __fadd_rn(cum, a.x); cum = __fadd_rn(cum, a.y); cum = __fadd_rn(cum, a.z); cum = __fadd_rn(cum, a.w);
                cum = __fadd_rn(cum, b.x); cum = __fadd_rn(cum, b.y); cum = __fadd_rn(cum, b.z); cum = __fadd_rn(cum, b.w);
            }
            for (; k < m; k++) cum = __fadd_rn(cum, x[k]);
        }
        __syncthreads();
    }
    if (tid == 0) out[0] = cum;
}

// batch rows of one round: states and action ids of the sampled slots
__global__ void k_rf_gather(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, const RfCall *__restrict__ call,
                            const int *__restrict__ round_idx, int B, float *__restrict__ S, int32_t *__restrict__ act) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    const uint32_t *r = records + (size_t)call->slots[(size_t)(*round_idx) * B + w] * L.record_words;
    for (int p = lane; p < obs; p += 32) S[(size_t)w * obs + p] = __uint_as_float(r[L.off_state + p]);
    if (lane == 0) act[w] = (int32_t)r[L.off_action];
}

// Both losses of a round, one CTA, fixed order.  Actor (reinforce.py:146-167): p = softmax(logits) over every action,
// nlp_j = -log(p_j[a_j] + 1e-8), loss = B * sum_j nlp_j (R - v_j) (the reference's B x B broadcast), dL/dnlp_j = B (R - v_j),
// softmax backward as torch evaluates it.  Critic (critic_utils.py:139-167): mean((v - R)^2), dv = 2 (v - R) / B.
__global__ void __launch_bounds__(256) k_rf_loss(int B, int A, const float *__restrict__ logits, const int32_t *__restrict__ act,
                                                 const float *__restrict__ v, float *__restrict__ dlogits, float *__restrict__ dv,
                                                 const RfCall *__restrict__ call, const int *__restrict__ round_idx) {
    __shared__ float red[256], red2[256];
    const float R = *call->ret, fb = (float)B, ib = 1.f / fb;
    float la = 0.f, lc = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const RowSoftmax sm(logits + (size_t)b * A, A);
        const int a = act[b];
        const float pa = sm(a), adv = R - v[b];
        la += -logf(pa + 1e-8f) * adv;
        const float g = -(__fmul_rn(adv, fb) / (pa + 1e-8f));       // dL/dp_a: log backward, then neg
        const float gp = g * pa;                                       // sum_k dL/dp_k p_k
        for (int k = 0; k < A; k++) dlogits[(size_t)b * A + k] = sm(k) * ((k == a ? g : 0.f) - gp);
        const float e = v[b] - R;
        lc += e * e;
        dv[b] = 2.f * e * ib;
    }
    red[threadIdx.x] = la; red2[threadIdx.x] = lc;
    __syncthreads();
    for (int o = 128; o; o >>= 1) {
        if (threadIdx.x < o) { red[threadIdx.x] += red[threadIdx.x + o]; red2[threadIdx.x] += red2[threadIdx.x + o]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        call->out_actor[*round_idx] = red[0] * fb;
        call->out_critic[*round_idx] = red2[0] * ib;
    }
}

__global__ void k_rf_bump(int *round_idx) { *round_idx += 1; }

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_reinforce {
    prl_reinforce_cfg cfg;
    Mlp2 an, cn;          // actor (softmax head) and critic (scalar head) layouts
    float *actor, *actor_m, *actor_v, *actor_x, *critic, *critic_m, *critic_v, *critic_x;
    int64_t adam_step;
    // workspace
    float *S, *ah1, *ah2, *logits, *ch1, *ch2, *v, *dlogits, *dv, *dh2, *dh1, *g_actor, *g_critic, *boot;
    int32_t *act, *slots, *logical;
    float2 *scal_a, *scal_c;
    RfCall *call;
    int *round_idx;
    Stage stage;
    bool use_graph;
    cudaGraphExec_t graph_exec;
    int graph_batch;
    const uint32_t *graph_buf;
    int launches_per_round;
    int64_t last_launches;
};

static int rf_check(const prl_reinforce_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->actor_h1 > 0 && c->actor_h2 > 0 && c->critic_h1 > 0 && c->critic_h2 > 0, "dimensions must be positive");
    PRL_REQUIRE(c->n_actions > 0 && c->n_actions <= kMaxA, "n_actions must be in [1, 255]");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    return PRL_OK;
}
static void rf_layout(prl_reinforce *s) {
    const prl_reinforce_cfg &c = s->cfg;
    s->an = mlp2(c.obs_dim, c.actor_h1, c.actor_h2, c.n_actions);
    s->cn = mlp2(c.obs_dim, c.critic_h1, c.critic_h2, 1);
}
extern "C" int64_t prl_reinforce_actor_param_count(const prl_reinforce_cfg *c) {
    if (rf_check(c)) return -1;
    prl_reinforce t; t.cfg = *c; rf_layout(&t);
    return t.an.P;
}
extern "C" int64_t prl_reinforce_critic_param_count(const prl_reinforce_cfg *c) {
    if (rf_check(c)) return -1;
    prl_reinforce t; t.cfg = *c; rf_layout(&t);
    return t.cn.P;
}
// the workspace, in order; base == null: only its size
static int64_t rf_carve(prl_reinforce *s, void *base) {
    const prl_reinforce_cfg &c = s->cfg;
    const int64_t B = c.max_batch, A = c.n_actions, O = c.obs_dim, MRB = (int64_t)c.max_rounds * c.max_batch;
    const int64_t hmax1 = c.actor_h1 > c.critic_h1 ? c.actor_h1 : c.critic_h1, hmax2 = c.actor_h2 > c.critic_h2 ? c.actor_h2 : c.critic_h2;
    Carve w{(char *)base};
    w(s->S, B * O); w(s->ah1, B * c.actor_h1); w(s->ah2, B * c.actor_h2); w(s->logits, B * A);
    w(s->ch1, B * c.critic_h1); w(s->ch2, B * c.critic_h2); w(s->v, B); w(s->dlogits, B * A); w(s->dv, B);
    w(s->dh2, B * hmax2); w(s->dh1, B * hmax1); w(s->g_actor, s->an.P); w(s->g_critic, s->cn.P);
    w(s->boot, 64);
    w(s->act, B); w(s->slots, MRB); w(s->logical, MRB);
    w(s->scal_a, 2 * (int64_t)c.max_rounds + 32);                                        // scal_a | scal_c | call | round_idx
    return w.bytes;
}
extern "C" int64_t prl_reinforce_workspace_bytes(const prl_reinforce_cfg *c) {
    if (rf_check(c)) return -1;
    prl_reinforce t; t.cfg = *c; rf_layout(&t);
    return rf_carve(&t, nullptr);
}
extern "C" int prl_reinforce_create(prl_reinforce **out, const prl_reinforce_cfg *cfg, float *actor_w, float *actor_m, float *actor_v,
                                    float *actor_vmax, float *critic_w, float *critic_m, float *critic_v, float *critic_vmax,
                                    int64_t adam_step, void *workspace) {
    PRL_REQUIRE(out && actor_w && actor_m && actor_v && actor_vmax && critic_w && critic_m && critic_v && critic_vmax && workspace,
                "null argument");
    int rc = rf_check(cfg);
    if (rc) return rc;
    prl_reinforce *s = new (std::nothrow) prl_reinforce();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    rf_layout(s);
    s->actor = actor_w; s->actor_m = actor_m; s->actor_v = actor_v; s->actor_x = actor_vmax;
    s->critic = critic_w; s->critic_m = critic_m; s->critic_v = critic_v; s->critic_x = critic_vmax;
    s->adam_step = adam_step;
    rf_carve(s, workspace);
    s->scal_c = s->scal_a + cfg->max_rounds;
    s->call = (RfCall *)(s->scal_c + cfg->max_rounds); s->round_idx = (int *)(s->call + 1);
    static_assert(sizeof(RfCall) + 4 <= 32 * 8, "call block fits the reserved tail");
    s->use_graph = true; s->graph_exec = nullptr; s->graph_batch = 0; s->graph_buf = nullptr; s->last_launches = 0;
    s->launches_per_round = 0;
    cudaError_t e = s->stage.open((size_t)cfg->max_rounds * 16 + 256);
    if (e != cudaSuccess) { delete s; return fail(PRL_ECUDA, "prl_reinforce_create: %s", cudaGetErrorString(e)); }
    *out = s;
    return PRL_OK;
}
extern "C" int prl_reinforce_destroy(prl_reinforce *s) {
    if (!s) return PRL_OK;
    s->stage.close();
    if (s->graph_exec) cudaGraphExecDestroy(s->graph_exec);
    delete s;
    return PRL_OK;
}
extern "C" int64_t prl_reinforce_adam_step(const prl_reinforce *s) { return s ? s->adam_step : -1; }
extern "C" int prl_reinforce_set_lr(prl_reinforce *s, double actor_lr, double critic_lr) {
    PRL_REQUIRE(s, "null handle");
    PRL_REQUIRE(actor_lr >= 0.0 && critic_lr >= 0.0, "learning rates must be non-negative");
    s->cfg.actor_lr = actor_lr;
    s->cfg.critic_lr = critic_lr;
    return PRL_OK;
}
extern "C" int prl_reinforce_set_graph(prl_reinforce *s, int enable) {
    PRL_REQUIRE(s, "null handle");
    s->use_graph = enable != 0;
    return PRL_OK;
}
extern "C" int64_t prl_reinforce_last_launches(const prl_reinforce *s) { return s ? s->last_launches : -1; }

static int rf_buffer_ok(const prl_reinforce *s, const prl_buf *buf) {
    const prl_reinforce_cfg &c = s->cfg;
    PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.obs_dim == c.obs_dim && buf->desc.n_actions == c.n_actions,
                "REINFORCE needs a discrete-action buffer with matching obs_dim / n_actions");
    PRL_REQUIRE(buf->shard_world <= 1, "the buffer is one shard of a multi-GPU buffer: REINFORCE reads local buffers only");
    return PRL_OK;
}

// REINFORCE.learn's return pass (reinforce.py:179-201): out_return_dev f32[2] = {R, critic(s'_newest) * (1 - terminated)}
extern "C" int prl_reinforce_returns(prl_reinforce *s, prl_buf *buf, float *out_return_dev, void *stream_) {
    PRL_REQUIRE(s && buf && out_return_dev, "null argument");
    int rc = rf_buffer_ok(s, buf);
    if (rc) return rc;
    const int64_t n = buf->len;
    PRL_REQUIRE(n > 0, "empty buffer (reference: assert len(replay_buffer.memory) > 0)");
    cudaStream_t st = (cudaStream_t)stream_;
    const int64_t cap = buf->desc.capacity, head = (buf->write_pos - n + cap) % cap;
    GemmLauncher L; L.st = st;
    k_last_next_state<<<1, 128, 0, st>>>(buf->records, buf->lay, s->cfg.obs_dim, (head + n - 1) % cap, s->S);
    mlp2_forward(L, s->cn, s->critic, s->S, 1, s->ch1, s->ch2, s->boot);
    k_rf_fold<<<1, 256, 0, st>>>(buf->records, buf->lay, head, cap, n, s->boot, out_return_dev);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

// one learner round, launched (or captured) on `st`; everything round- or call-dependent is read through s->call / s->round_idx
static int rf_round(prl_reinforce *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_reinforce_cfg &c = s->cfg;
    // the decay factors are overridden by call->decay_a / decay_c (k_adamw's decay pointer)
    const AdamHp h = adam_hp(0.0, c.beta1, c.beta2, c.eps, c.weight_decay);
    GemmLauncher L; L.st = st;
    const int eb = 256;
    k_rf_gather<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf->records, buf->lay, c.obs_dim, s->call, s->round_idx, B, s->S, s->act);
    mlp2_forward(L, s->cn, s->critic, s->S, B, s->ch1, s->ch2, s->v);
    mlp2_forward(L, s->an, s->actor, s->S, B, s->ah1, s->ah2, s->logits);
    k_rf_loss<<<1, 256, 0, st>>>(B, c.n_actions, s->logits, s->act, s->v, s->dlogits, s->dv, s->call, s->round_idx);
    // ---------------- actor step (actor_critic_base.py:333-343)
    mlp2_backward(L, s->an, s->actor, s->g_actor, s->dlogits, s->S, s->ah1, s->ah2, s->dh2, s->dh1, B);
    k_adamw<<<(s->an.P + eb - 1) / eb, eb, 0, st>>>(s->an.P, s->actor, s->actor_m, s->actor_v, s->actor_x, s->g_actor, h, s->scal_a,
                                                  s->round_idx, nullptr, 0.f, 0.f, &s->call->decay_a);
    // ---------------- critic step (actor_critic_base.py:344-349), same v: the critic has not changed
    mlp2_backward(L, s->cn, s->critic, s->g_critic, s->dv, s->S, s->ch1, s->ch2, s->dh2, s->dh1, B);   // + one k_head_bwd
    k_adamw<<<(s->cn.P + eb - 1) / eb, eb, 0, st>>>(s->cn.P, s->critic, s->critic_m, s->critic_v, s->critic_x, s->g_critic, h, s->scal_c,
                                                  s->round_idx, nullptr, 0.f, 0.f, &s->call->decay_c);
    k_rf_bump<<<1, 1, 0, st>>>(s->round_idx);
    s->launches_per_round = L.count + 6;   // gather, loss, head backward, 2 x adamw, round counter
    return PRL_OK;
}

// PolicyLearner.learn (policy_learner.py:162-204) over a buffer whose return R the last prl_reinforce_returns wrote to
// return_dev[0]: rounds x (sample -> actor step -> critic step)
extern "C" int prl_reinforce_learn(prl_reinforce *s, prl_buf *buf, int rounds, int batch, const float *return_dev, float *out_actor_loss,
                                   float *out_critic_loss, int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && return_dev && out_actor_loss && out_critic_loss, "null argument");
    const prl_reinforce_cfg &c = s->cfg;
    PRL_REQUIRE(rounds > 0 && rounds <= c.max_rounds && batch > 0 && batch <= c.max_batch, "rounds / batch outside the configured maxima");
    int rc = rf_buffer_ok(s, buf);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream_;
    rc = prl_buf_sample_indices(buf, rounds, batch, out_logical ? out_logical : s->logical, s->slots, stream_);
    if (rc) return rc;
    // per-call block: Adam scalars of every round (as torch evaluates them in double), decay factors, pointers
    float2 *hs;
    rc = s->stage.wait(&hs);
    if (rc) return rc;
    const int MR = c.max_rounds;
    for (int r = 0; r < rounds; r++) {
        hs[r] = adam_scal(c.actor_lr, c.beta1, c.beta2, s->adam_step + r + 1);
        hs[MR + r] = adam_scal(c.critic_lr, c.beta1, c.beta2, s->adam_step + r + 1);
    }
    RfCall *hc = reinterpret_cast<RfCall *>(hs + 2 * (size_t)MR);
    hc->slots = s->slots; hc->ret = return_dev; hc->out_actor = out_actor_loss; hc->out_critic = out_critic_loss;
    hc->decay_a = (float)(1.0 - c.actor_lr * c.weight_decay);
    hc->decay_c = (float)(1.0 - c.critic_lr * c.weight_decay);
    *reinterpret_cast<int *>(hc + 1) = 0;
    // scal_a | scal_c | call | round_idx are contiguous on the device in the same order
    rc = s->stage.send(s->scal_a, 2 * (size_t)MR * 8 + sizeof(RfCall) + 4, st);
    if (rc) return rc;
    if (s->use_graph) {
        if (!s->graph_exec || s->graph_batch != batch || s->graph_buf != buf->records) {
            rc = capture_graph(&s->graph_exec, "prl_reinforce_learn", [&](cudaStream_t cs) { return rf_round(s, buf, batch, cs); });
            if (rc) return rc;
            s->graph_batch = batch; s->graph_buf = buf->records;
        }
        for (int r = 0; r < rounds; r++) PRL_CUDA(cudaGraphLaunch(s->graph_exec, st));
    } else {
        for (int r = 0; r < rounds; r++) {
            rc = rf_round(s, buf, batch, st);
            if (rc) return rc;
        }
    }
    PRL_CUDA(cudaGetLastError());
    s->adam_step += rounds;
    s->last_launches = (int64_t)s->launches_per_round * rounds;
    return PRL_OK;
}
