// ppo.cu — K7: generalized advantage estimation + truncated lambda returns over a rollout.
//
// Replaces the per-transition Python loop of ProximalPolicyOptimization.preprocess_replay_buffer
// (pearl/policy_learners/sequential_decision_making/ppo.py:271-293), which walks the stored
// transitions newest -> oldest:
//     td    = reward + gamma * next_value * (~terminated) - V[i]
//     gae   = td + gamma * lambda * (not (terminated or truncated)) * gae
//     lam_return = gae + V[i];   next_value = V[i]
// (next_value starts as the critic's value of the LAST stored next_state; note that V(s_{t+1}) is
// taken to be the value of the next STORED transition's state — a reference quirk that is mirrored.)
//
// td depends only on the transition and its newer neighbour, and the gae chain restarts at every
// terminated / truncated transition, so each chain (one episode) is walked sequentially by one
// thread with exactly the reference's fp32 operation order => results are BIT-IDENTICAL to the
// reference loop, while the episodes of the rollout run in parallel.  HBM traffic: 10 bytes read +
// 8 bytes written per transition.
#include <stdarg.h>

#include "common.cuh"

using namespace prl;

namespace {

// arrays are in TIME order (index 0 = oldest stored transition)
// A chain = an episode segment; its newest element ("head") is the last stored transition or one with terminated /
// truncated set.  k_ppo_gae_heads compacts the head positions (order irrelevant: chains are independent); k_ppo_gae then
// gives a CTA 32 chains at a time and moves them newest -> oldest in blocks of 64 transitions:
//   A  all four warps: a chain's block is 256 contiguous bytes per array, so every global access is coalesced; the
//      temporal-difference term td (it depends only on a transition and its newer neighbour) is computed here, in the
//      reference's fp32 operation order, and staged in shared memory with the chain-end flags;
//   B  warp 0, one lane per chain: the dependent recurrence gae = td + c * gae over the 64 staged values (two flops per
//      transition on the serial path, four transitions per flag word), results written back in place;
//   C  all four warps: coalesced stores of gae and gae + V.
// Results are bit-identical to the Python loop (ppo.py:271-293).  History: round 1 let the head's own thread of a
// one-thread-per-transition grid walk the chain (one active lane per warp, 0.04 of the HBM roofline at 16M transitions);
// a chain per THREAD with register prefetch reached 0.14: 32 lanes 2 KB apart make every access a lone 32-byte sector.
constexpr int kGaeBlk = 64;

__global__ void k_ppo_gae_heads(int n, const uint8_t *__restrict__ terminated, const uint8_t *__restrict__ truncated,
                                int *__restrict__ heads, int *__restrict__ count) {
    // four transitions per thread (one flag word per array when the arrays are word-aligned)
    const int q = blockIdx.x * blockDim.x + threadIdx.x, t0 = q * 4, lane = threadIdx.x & 31;
    const bool aligned = ((reinterpret_cast<uintptr_t>(terminated) | reinterpret_cast<uintptr_t>(truncated)) & 3) == 0;
    uint32_t f = 0;
    if (t0 + 3 < n && aligned) {
        f = *reinterpret_cast<const uint32_t *>(terminated + t0) | *reinterpret_cast<const uint32_t *>(truncated + t0);
    } else {
        for (int u = 0; u < 4; u++)
            if (t0 + u < n && (terminated[t0 + u] | truncated[t0 + u])) f |= 0xffu << (8 * u);
    }
    unsigned mask = 0;
#pragma unroll
    for (int u = 0; u < 4; u++)
        if (t0 + u < n && (((f >> (8 * u)) & 0xffu) != 0 || t0 + u == n - 1)) mask |= 1u << u;
    const int mine = __popc(mask);
    int incl = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
    }
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    int base = 0;
    if (lane == 31 && total) base = atomicAdd(count, total);
    base = __shfl_sync(0xffffffffu, base, 31) + incl - mine;
#pragma unroll
    for (int u = 0; u < 4; u++)
        if (mask & (1u << u)) heads[base++] = t0 + u;
}

__global__ void __launch_bounds__(128) k_ppo_gae(int n, const int *__restrict__ heads, const int *__restrict__ count, const float *__restrict__ values,
                          float last_next_value_host, const float *__restrict__ last_next_value_dev, float incoming_gae,
                          const float *__restrict__ reward, const uint8_t *__restrict__ terminated, const uint8_t *__restrict__ truncated,
                          float gamma, float c_live, float *__restrict__ out_gae, float *__restrict__ out_lam_return) {
    __shared__ float s_td[32][kGaeBlk + 1], s_v[32][kGaeBlk + 1];
    __shared__ __align__(4) uint8_t s_cut[32][kGaeBlk + 4];
    __shared__ int s_top[32], s_len[32], s_any;
    const int nh = *count, tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
    const float last_next_value = last_next_value_dev ? *last_next_value_dev : last_next_value_host;
    for (int g0 = blockIdx.x * 32; g0 < nh; g0 += gridDim.x * 32) {
        // chain state lives in warp 0, lane = chain
        int top = -1;
        float gae = 0.f;
        bool first = true;
        if (w == 0) {
            if (g0 + lane < nh) top = heads[g0 + lane];
            // the chain headed by the newest element continues a chain of NEWER transitions held elsewhere (a later time
            // shard): it starts from that chain's gae instead of 0 (multiplied by 0 below if the newest element ends an episode)
            if (top == n - 1) gae = incoming_gae;
            s_top[lane] = top;
        }
        __syncthreads();
        while (true) {
            // ---- A: stage td, V and the chain-end flags of every live chain's next block.  All of a warp's loads for
            //         four chains are issued before any is used (one memory round trip per four chains, not per chain)
#pragma unroll 1
            for (int jb = 0; jb < 8; jb += 4) {
                float v[4][kGaeBlk / 32], r[4][kGaeBlk / 32], nv[4][kGaeBlk / 32];
                uint8_t te[4][kGaeBlk / 32], tr[4][kGaeBlk / 32];
                int tjs[4];
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const int tj = s_top[w + 4 * (jb + q)];
                    tjs[q] = tj;
#pragma unroll
                    for (int e = 0; e < kGaeBlk / 32; e++) {
                        const int idx = tj - lane - 32 * e;
                        const bool ok = tj >= 0 && idx >= 0;
                        const int ia = ok ? idx : 0, ib = (ok && idx + 1 < n) ? idx + 1 : 0;
                        v[q][e] = values[ia]; r[q][e] = reward[ia]; nv[q][e] = values[ib];
                        te[q][e] = terminated[ia]; tr[q][e] = truncated[ia];
                    }
                }
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const int j = w + 4 * (jb + q), tj = tjs[q];
                    if (tj < 0) continue;
#pragma unroll
                    for (int e = 0; e < kGaeBlk / 32; e++) {
                        const int k = lane + 32 * e, idx = tj - k;
                        float td = 0.f;
                        uint8_t cut = 1;                                // below the oldest transition: stops the walk
                        if (idx >= 0) {
                            const float nvx = idx + 1 < n ? nv[q][e] : last_next_value;   // the next STORED transition's value
                            const bool term = te[q][e] != 0;
                            cut = (term || tr[q][e] != 0) ? 1 : 0;
                            // reward + gamma * next_value * (~terminated) - V[i]   (left to right, fp32)
                            td = __fsub_rn(__fadd_rn(r[q][e], __fmul_rn(__fmul_rn(gamma, nvx), term ? 0.f : 1.f)), v[q][e]);
                        }
                        s_td[j][k] = td;
                        s_v[j][k] = v[q][e];
                        s_cut[j][k] = cut;
                    }
                }
            }
            __syncthreads();
            // ---- B: the recurrence, one lane per chain:  gae = td + (gamma * lambda * mask) * gae
            //         (the scalar product gamma * lambda is evaluated in double by Python and passed in as c_live)
            int next_top = -1;
            if (w == 0 && top >= 0) {
                int k = 0;
                bool ended = false;
                for (; k < kGaeBlk && !ended; k += 4) {
                    const uint32_t cw = *reinterpret_cast<const uint32_t *>(&s_cut[lane][k]);
                    const float t0 = s_td[lane][k], t1 = s_td[lane][k + 1], t2 = s_td[lane][k + 2], t3 = s_td[lane][k + 3];
                    if (cw == 0) {                                     // no episode end among these four
                        const float g0v = __fadd_rn(t0, __fmul_rn(c_live, gae));
                        const float g1v = __fadd_rn(t1, __fmul_rn(c_live, g0v));
                        const float g2v = __fadd_rn(t2, __fmul_rn(c_live, g1v));
                        gae = __fadd_rn(t3, __fmul_rn(c_live, g2v));
                        s_td[lane][k] = g0v; s_td[lane][k + 1] = g1v; s_td[lane][k + 2] = g2v; s_td[lane][k + 3] = gae;
                        continue;
                    }
                    const float tt[4] = {t0, t1, t2, t3};
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        if (ended) break;
                        const bool cut = ((cw >> (8 * u)) & 0xffu) != 0;
                        float mult = c_live;
                        if (first && k + u == 0) mult = cut ? 0.f : c_live;   // the head itself
                        else if (cut) { ended = true; s_len[lane] = k + u; break; }   // the next chain's head
                        gae = __fadd_rn(tt[u], __fmul_rn(mult, gae));
                        s_td[lane][k + u] = gae;
                    }
                }
                first = false;
                if (!ended) { s_len[lane] = kGaeBlk; next_top = top - kGaeBlk; }
            }
            __syncthreads();
            // ---- C: coalesced stores
#pragma unroll 2
            for (int jj = 0; jj < 8; jj++) {
                const int j = w + 4 * jj, tj = s_top[j];
                if (tj < 0) continue;
                const int len = s_len[j];
#pragma unroll
                for (int e = 0; e < kGaeBlk / 32; e++) {
                    const int k = lane + 32 * e;
                    if (k < len) {
                        const float g = s_td[j][k];
                        out_gae[tj - k] = g;
                        out_lam_return[tj - k] = __fadd_rn(g, s_v[j][k]);
                    }
                }
            }
            __syncthreads();
            if (w == 0) {
                top = next_top;
                s_top[lane] = top;
                const unsigned live = __ballot_sync(0xffffffffu, top >= 0);
                if (lane == 0) s_any = live != 0;
            }
            __syncthreads();
            if (!s_any) break;
        }
    }
}

}  // namespace

// heads: int32[n] scratch, count: int32[1] scratch (both device)
static int launch_gae(int n, const float *values, float last_next_value, const float *last_next_value_dev, float incoming_gae,
                      const float *reward, const uint8_t *term, const uint8_t *trunc, float gamma, float c_live, float *out_gae,
                      float *out_lam_return, int *heads, int *count, cudaStream_t st) {
    PRL_CUDA(cudaMemsetAsync(count, 0, sizeof(int), st));
    k_ppo_gae_heads<<<((n + 3) / 4 + 255) / 256, 256, 0, st>>>(n, term, trunc, heads, count);
    const int groups = (n + 31) / 32;                              // an upper bound on chains / 32 (the count is on the device)
    const int blocks = groups < 148 * 16 ? groups : 148 * 16;
    k_ppo_gae<<<blocks, 128, 0, st>>>(n, heads, count, values, last_next_value, last_next_value_dev, incoming_gae, reward, term, trunc, gamma,
                                      c_live, out_gae, out_lam_return);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

extern "C" int prl_ppo_gae(int n, const float *values_dev, float last_next_value, const float *reward_dev,
                           const uint8_t *terminated_dev, const uint8_t *truncated_dev, double gamma, double lam,
                           float *out_gae_dev, float *out_lam_return_dev, int32_t *scratch_dev, void *stream) {
    PRL_REQUIRE(n >= 0, "negative length");
    if (n == 0) return PRL_OK;
    PRL_REQUIRE(values_dev && reward_dev && terminated_dev && truncated_dev && out_gae_dev && out_lam_return_dev && scratch_dev,
                "null argument");
    return launch_gae(n, values_dev, last_next_value, nullptr, 0.f, reward_dev, terminated_dev, truncated_dev, (float)gamma,
                      (float)(gamma * lam), out_gae_dev, out_lam_return_dev, scratch_dev + 1, scratch_dev, (cudaStream_t)stream);
}

// ====================================================================================================
// PPO learner: ProximalPolicyOptimization.learn (ppo.py:195-293 preprocess, :152-193 losses) on top of
// ActorCriticBase.learn_batch (actor_critic_base.py:309-349) and PolicyLearner.learn
// (policy_learner.py:162-204).  VanillaActorNetwork (softmax policy, actor_networks.py:107-176) and
// VanillaValueNetwork, two hidden layers each; three AdamW(amsgrad) steps per round are two here
// (actor, critic).  Same launch structure as the SAC learner (gemm.cuh + small kernels, CUDA-graph replay).
// ====================================================================================================
#include <math.h>

#include <new>

#include "ac_nets.cuh"
#include "rounds.cuh"

namespace {

struct PpoCall {
    const int32_t *logical, *slots;   // [rounds][B]
    const float *gae, *lam_return, *old_probs;   // [len] in time order
    float *out_actor, *out_critic;
};

// rollout rows [i0, i0 + rows) in time order -> contiguous states / action ids (+ reward / flags for the whole rollout)
__global__ void k_ppo_rollout_rows(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int64_t head, int64_t cap, int64_t i0,
                                   int rows, float *__restrict__ S, int32_t *__restrict__ act, float *__restrict__ reward,
                                   uint8_t *__restrict__ term, uint8_t *__restrict__ trunc) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= rows) return;
    const uint32_t *r = records + (size_t)((head + i0 + w) % cap) * L.record_words;
    for (int p = lane; p < obs; p += 32) S[(size_t)w * obs + p] = __uint_as_float(r[L.off_state + p]);
    if (lane == 0) {
        act[w] = (int32_t)r[L.off_action];
        reward[i0 + w] = __uint_as_float(r[L.off_reward]);
        const uint32_t f = r[L.off_flags];
        term[i0 + w] = f & 1u; trunc[i0 + w] = (f >> 1) & 1u;
    }
}
// probability of the taken action under softmax(logits)
__global__ void k_ppo_taken_prob(int rows, int A, const float *__restrict__ logits, const int32_t *__restrict__ act, float *__restrict__ out) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= rows) return;
    const RowSoftmax sm(logits + (size_t)b * A, A);
    out[b] = sm(act[b]);
}
// batch rows of one round
__global__ void k_ppo_gather(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, const PpoCall *__restrict__ call,
                             const int *__restrict__ round_idx, int B, float *__restrict__ S, int32_t *__restrict__ act, float *__restrict__ gae,
                             float *__restrict__ lam, float *__restrict__ old) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= B) return;
    const size_t o = (size_t)(*round_idx) * B + w;
    const uint32_t *r = records + (size_t)call->slots[o] * L.record_words;
    for (int p = lane; p < obs; p += 32) S[(size_t)w * obs + p] = __uint_as_float(r[L.off_state + p]);
    if (lane == 0) {
        const int i = call->logical[o];
        act[w] = (int32_t)r[L.off_action];
        gae[w] = call->gae[i]; lam[w] = call->lam_return[i]; old[w] = call->old_probs[i];
    }
}
// clipped surrogate (ppo.py:152-184): loss = sum(-min(r * gae, clamp(r) * gae)) - beta * H(Categorical(ap)), and dLoss/dlogits
__global__ void k_ppo_actor_loss(int B, int A, const float *__restrict__ logits, const int32_t *__restrict__ act, const float *__restrict__ gae,
                                 const float *__restrict__ old, float eps_clip, float beta, float *__restrict__ ap_buf,
                                 float *__restrict__ dlogits, const PpoCall *__restrict__ call, const int *__restrict__ round_idx) {
    __shared__ float red[256], red2[256];
    float loss = 0.f, psum = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const RowSoftmax sm(logits + (size_t)b * A, A);
        const int a = act[b];
        const float ap = sm(a);
        const float r = ap / old[b], g = gae[b];
        const float lo = 1.f - eps_clip, hi = 1.f + eps_clip;
        const float clip = fminf(fmaxf(r, lo), hi);
        const float x1 = r * g, x2 = clip * g;
        loss += -fminf(x1, x2);
        // torch.min splits ties evenly; clamp passes the gradient inside [lo, hi] (ends included)
        const float inside = (r >= lo && r <= hi) ? 1.f : 0.f;
        const float w1 = x1 < x2 ? 1.f : (x1 == x2 ? 0.5f : 0.f), w2 = 1.f - w1;
        const float dr = -g * (w1 + w2 * inside);
        const float dap = dr / old[b];
        for (int j = 0; j < A; j++) {
            const float pj = sm(j);
            dlogits[(size_t)b * A + j] = dap * ap * ((j == a ? 1.f : 0.f) - pj);
        }
        ap_buf[b] = ap;
        psum += ap;
    }
    red[threadIdx.x] = loss; red2[threadIdx.x] = psum;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) { red[threadIdx.x] += red[threadIdx.x + o]; red2[threadIdx.x] += red2[threadIdx.x + o]; } __syncthreads(); }
    const float total = red[0], ptot = red2[0];
    __syncthreads();
    // entropy of Categorical(probs = ap / sum(ap)) as torch evaluates it (probs clamped to [eps, 1 - eps] inside the log)
    float ent = 0.f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float p = ap_buf[b] / ptot;
        ent += p * logf(fminf(fmaxf(p, 1.1920929e-07f), 1.f - 1.1920929e-07f));
    }
    red[threadIdx.x] = ent;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) call->out_actor[*round_idx] = total - beta * (-red[0]);
}
// MSE(v, lam_return): loss and dLoss/dv; advances the round counter (last kernel of the round reads it before)
__global__ void k_ppo_critic_loss(int B, const float *__restrict__ v, const float *__restrict__ target, float *__restrict__ dv,
                                  const PpoCall *__restrict__ call, const int *__restrict__ round_idx) {
    __shared__ float red[256];
    float s = 0.f;
    const float ib = 1.f / (float)B;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        const float e = v[b] - target[b];
        s += e * e;
        dv[b] = 2.f * e * ib;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) call->out_critic[*round_idx] = red[0] * ib;
}
__global__ void k_ppo_bump(int *round_idx) { *round_idx += 1; }
__global__ void k_ppo_cuts(int n, const uint8_t *__restrict__ term, const uint8_t *__restrict__ trunc, uint8_t *__restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (term[i] | trunc[i]) ? 1 : 0;
}

}  // namespace

struct prl_ppo : Rounds<prl_ppo, PpoCall> {
    static constexpr const char *kFn = "prl_ppo";
    static constexpr int kScal = 2;   // actor, critic
    prl_ppo_cfg cfg;
    Mlp2 an, cn;          // actor (softmax head) and critic (scalar head) layouts
    float *actor, *actor_m, *actor_v, *actor_x, *critic, *critic_m, *critic_v, *critic_x;
    // workspace
    float *S, *h1, *h2, *logits, *v, *gae, *lam, *old, *ap, *dlogits, *dh2, *dh1, *dv, *g_actor, *g_critic, *reward, *last_value;
    int32_t *act;
    uint8_t *term, *trunc;
    int *gae_heads;           // [1 + max_rollout]: count, then the chain-head positions of the GAE pass
    int64_t pre_n;      // rollout length of the last prl_ppo_preprocess
    double &lr(int k) { return k == 0 ? cfg.actor_lr : cfg.critic_lr; }
    int buffer_ok(const prl_buf *buf) const {
        PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.obs_dim == cfg.obs_dim && buf->desc.n_actions == cfg.n_actions,
                    "PPO needs a discrete-action buffer with matching dimensions");
        return PRL_OK;
    }
    static int round(prl_ppo *s, prl_buf *buf, int B, cudaStream_t st);
};

// rollout rows evaluated per pass of the preprocessing: the whole rollout when it fits 65536 rows (a pass is 8 launches,
// and at 8192 rows per pass the 64k-step rollout of the benchmark spent more time between launches than in them)
static inline int64_t ppo_chunk(const prl_ppo_cfg *c) {
    const int64_t r = c->max_rollout < 65536 ? c->max_rollout : 65536;
    return r < 8192 ? 8192 : r;
}

static int ppo_check(const prl_ppo_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->n_actions > 0 && c->actor_h1 > 0 && c->actor_h2 > 0 && c->critic_h1 > 0 && c->critic_h2 > 0,
                "dimensions must be positive");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0 && c->max_rollout > 0, "max_batch / max_rounds / max_rollout must be positive");
    return PRL_OK;
}
static void ppo_layout(prl_ppo *s) {
    const prl_ppo_cfg &c = s->cfg;
    s->an = mlp2(c.obs_dim, c.actor_h1, c.actor_h2, c.n_actions);
    s->cn = mlp2(c.obs_dim, c.critic_h1, c.critic_h2, 1);
}
extern "C" int64_t prl_ppo_actor_param_count(const prl_ppo_cfg *c) {
    if (ppo_check(c)) return -1;
    prl_ppo t; t.cfg = *c; ppo_layout(&t);
    return t.an.P;
}
extern "C" int64_t prl_ppo_critic_param_count(const prl_ppo_cfg *c) {
    if (ppo_check(c)) return -1;
    prl_ppo t; t.cfg = *c; ppo_layout(&t);
    return t.cn.P;
}
// the workspace, in order; base == null: only its size
static int64_t ppo_carve(prl_ppo *s, void *base) {
    const prl_ppo_cfg &c = s->cfg;
    const int64_t R = c.max_batch > ppo_chunk(&c) ? c.max_batch : ppo_chunk(&c);   // rows of the widest pass
    const int64_t hmax1 = c.actor_h1 > c.critic_h1 ? c.actor_h1 : c.critic_h1, hmax2 = c.actor_h2 > c.critic_h2 ? c.actor_h2 : c.critic_h2;
    const int64_t A = c.n_actions;
    Carve w{(char *)base};
    w(s->S, R * c.obs_dim); w(s->h1, R * hmax1); w(s->h2, R * hmax2); w(s->logits, R * A); w(s->v, R);
    w(s->gae, R); w(s->lam, R); w(s->old, R); w(s->ap, R); w(s->dlogits, R * A);
    w(s->dh2, R * hmax2); w(s->dh1, R * hmax1); w(s->dv, R); w(s->g_actor, s->an.P); w(s->g_critic, s->cn.P);
    w(s->reward, c.max_rollout); w(s->last_value, 64);
    w(s->act, R);
    w(s->term, c.max_rollout); w(s->trunc, c.max_rollout);
    s->carve_tail(w, c.max_rounds, c.max_batch);
    w(s->gae_heads, c.max_rollout + 1);                                                  // count, then the GAE chain heads
    return w.bytes;
}
extern "C" int64_t prl_ppo_workspace_bytes(const prl_ppo_cfg *c) {
    if (ppo_check(c)) return -1;
    prl_ppo t; t.cfg = *c; ppo_layout(&t);
    return ppo_carve(&t, nullptr);
}
extern "C" int prl_ppo_create(prl_ppo **out, const prl_ppo_cfg *cfg, float *actor_w, float *actor_m, float *actor_v, float *actor_vmax,
                              float *critic_w, float *critic_m, float *critic_v, float *critic_vmax, int64_t adam_step, void *workspace) {
    PRL_REQUIRE(out && actor_w && actor_m && actor_v && actor_vmax && critic_w && critic_m && critic_v && critic_vmax && workspace,
                "null argument");
    int rc = ppo_check(cfg);
    if (rc) return rc;
    prl_ppo *s = new (std::nothrow) prl_ppo();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    ppo_layout(s);
    s->actor = actor_w; s->actor_m = actor_m; s->actor_v = actor_v; s->actor_x = actor_vmax;
    s->critic = critic_w; s->critic_m = critic_m; s->critic_v = critic_v; s->critic_x = critic_vmax;
    s->adam_step = adam_step;
    ppo_carve(s, workspace);
    return prl_ppo::open(s, out);
}
extern "C" int prl_ppo_destroy(prl_ppo *s) { return prl_ppo::destroy(s); }
extern "C" int64_t prl_ppo_adam_step(const prl_ppo *s) { return prl_ppo::adam_step_of(s); }
extern "C" int prl_ppo_set_graph(prl_ppo *s, int enable) { return prl_ppo::set_graph(s, enable); }
extern "C" int64_t prl_ppo_last_launches(const prl_ppo *s) { return prl_ppo::last_launches_of(s); }

static void ppo_actor_forward(prl_ppo *s, GemmLauncher &L, int rows) {
    mlp2_forward(L, s->an, s->actor, s->S, rows, s->h1, s->h2, s->logits);
}
static void ppo_critic_forward(prl_ppo *s, GemmLauncher &L, int rows, float *vout) {
    mlp2_forward(L, s->cn, s->critic, s->S, rows, s->h1, s->h2, vout);
}

// preprocess_replay_buffer (ppo.py:201-293): state values, taken-action probabilities, GAE and lambda returns of the whole
// rollout, in time order (index 0 = oldest stored transition)
extern "C" int prl_ppo_preprocess(prl_ppo *s, prl_buf *buf, float *out_values, float *out_action_probs, float *out_gae,
                                  float *out_lam_return, uint8_t *out_cut, void *stream_) {
    PRL_REQUIRE(s && buf && out_values && out_action_probs && out_gae && out_lam_return, "null argument");
    const prl_ppo_cfg &c = s->cfg;
    PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.obs_dim == c.obs_dim && buf->desc.n_actions == c.n_actions,
                "PPO needs a discrete-action buffer with matching dimensions");
    const int64_t n = buf->len;
    PRL_REQUIRE(n > 0, "empty rollout (reference: assert len(replay_buffer.memory) > 0)");
    PRL_REQUIRE(n <= c.max_rollout, "rollout longer than max_rollout");
    cudaStream_t st = (cudaStream_t)stream_;
    const int64_t cap = buf->desc.capacity, head = (buf->write_pos - buf->len + cap) % cap;
    GemmLauncher L; L.st = st;
    // a transition's value / action probability must not depend on how the rollout is cut into passes or time shards
    // (prl_ppo_gae_redo promises bit-identity with the unsharded rollout): one engine and one summation order for every pass
    L.fixed_order = true;
    L.engine = prl_get_contraction_engine() ? 2 : 0;
    const int64_t chunk = ppo_chunk(&c);
    for (int64_t i0 = 0; i0 < n; i0 += chunk) {
        const int rows = (int)((n - i0 < chunk) ? n - i0 : chunk);
        k_ppo_rollout_rows<<<(rows * 32 + 255) / 256, 256, 0, st>>>(buf->records, buf->lay, c.obs_dim, head, cap, i0, rows, s->S, s->act, s->reward,
                                                                  s->term, s->trunc);
        ppo_critic_forward(s, L, rows, out_values + i0);
        ppo_actor_forward(s, L, rows);
        k_ppo_taken_prob<<<(rows + 255) / 256, 256, 0, st>>>(rows, c.n_actions, s->logits, s->act, out_action_probs + i0);
    }
    k_last_next_state<<<1, 128, 0, st>>>(buf->records, buf->lay, c.obs_dim, (head + n - 1) % cap, s->S);
    ppo_critic_forward(s, L, 1, s->last_value);
    {
        const int rc = launch_gae((int)n, out_values, 0.f, s->last_value, 0.f, s->reward, s->term, s->trunc, (float)c.gamma,
                                  (float)(c.gamma * c.lam), out_gae, out_lam_return, s->gae_heads + 1, s->gae_heads, st);
        if (rc) return rc;
    }
    if (out_cut) k_ppo_cuts<<<(int)((n + 255) / 256), 256, 0, st>>>((int)n, s->term, s->trunc, out_cut);
    PRL_CUDA(cudaGetLastError());
    s->pre_n = n;
    return PRL_OK;
}

// A rollout sharded over ranks by contiguous time chunks (SURVEY.md 8e): the GAE recurrence of this chunk continues into
// the next (newer) chunk.  Re-run the chunk's chains with V(next) of its newest transition = the first state value of the
// next chunk and the chain entering from there = that chunk's first gae.  Same fp32 operation order as the unsharded
// kernel, so the sharded result is bit-identical to the whole rollout on one GPU.
extern "C" int prl_ppo_gae_redo(prl_ppo *s, const float *values_dev, float next_value, float incoming_gae, float *out_gae,
                                float *out_lam_return, void *stream_) {
    PRL_REQUIRE(s && values_dev && out_gae && out_lam_return, "null argument");
    PRL_REQUIRE(s->pre_n > 0, "prl_ppo_preprocess has not run on this handle");
    const prl_ppo_cfg &c = s->cfg;
    const int64_t n = s->pre_n;
    return launch_gae((int)n, values_dev, next_value, nullptr, incoming_gae, s->reward, s->term, s->trunc, (float)c.gamma,
                      (float)(c.gamma * c.lam), out_gae, out_lam_return, s->gae_heads + 1, s->gae_heads, (cudaStream_t)stream_);
}

int prl_ppo::round(prl_ppo *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_ppo_cfg &c = s->cfg;
    const float2 *scal_a = s->scal, *scal_c = s->scal + c.max_rounds;
    const int O = c.obs_dim;
    GemmLauncher L; L.st = st;
    const AdamHp ha = adam_hp(c.actor_lr, c.beta1, c.beta2, c.eps, c.weight_decay), hc = adam_hp(c.critic_lr, c.beta1, c.beta2, c.eps, c.weight_decay);
    const int eb = 256;
    k_ppo_gather<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf->records, buf->lay, O, s->call, s->round_idx, B, s->S, s->act, s->gae, s->lam, s->old);
    // ---------------- actor step
    ppo_actor_forward(s, L, B);
    k_ppo_actor_loss<<<1, 256, 0, st>>>(B, c.n_actions, s->logits, s->act, s->gae, s->old, (float)c.epsilon, (float)c.entropy_bonus, s->ap, s->dlogits,
                                        s->call, s->round_idx);
    mlp2_backward(L, s->an, s->actor, s->g_actor, s->dlogits, s->S, s->h1, s->h2, s->dh2, s->dh1, B);
    k_adamw<<<(s->an.P + eb - 1) / eb, eb, 0, st>>>(s->an.P, s->actor, s->actor_m, s->actor_v, s->actor_x, s->g_actor, ha, scal_a, s->round_idx,
                                                  nullptr, 0.f, 0.f);
    // ---------------- critic step (critic_utils.py:139-167)
    ppo_critic_forward(s, L, B, s->v);
    k_ppo_critic_loss<<<1, 256, 0, st>>>(B, s->v, s->lam, s->dv, s->call, s->round_idx);
    mlp2_backward(L, s->cn, s->critic, s->g_critic, s->dv, s->S, s->h1, s->h2, s->dh2, s->dh1, B);   // + one k_head_bwd
    k_adamw<<<(s->cn.P + eb - 1) / eb, eb, 0, st>>>(s->cn.P, s->critic, s->critic_m, s->critic_v, s->critic_x, s->g_critic, hc, scal_c,
                                                  s->round_idx, nullptr, 0.f, 0.f);
    k_ppo_bump<<<1, 1, 0, st>>>(s->round_idx);
    s->launches_per_round = L.count + 7;
    return PRL_OK;
}

// PolicyLearner.learn over the preprocessed rollout: rounds x (sample -> actor step -> critic step)
extern "C" int prl_ppo_learn(prl_ppo *s, prl_buf *buf, int rounds, int batch, const float *gae_dev, const float *lam_return_dev,
                             const float *action_probs_dev, float *out_actor_loss, float *out_critic_loss, int32_t *out_logical,
                             void *stream_) {
    PRL_REQUIRE(s && buf && gae_dev && lam_return_dev && action_probs_dev && out_actor_loss && out_critic_loss, "null argument");
    PpoCall call{};
    call.logical = out_logical ? out_logical : s->logical; call.gae = gae_dev; call.lam_return = lam_return_dev;
    call.old_probs = action_probs_dev; call.out_actor = out_actor_loss; call.out_critic = out_critic_loss;
    return prl_ppo::learn(s, buf, rounds, batch, 0, out_logical, call, stream_);
}
