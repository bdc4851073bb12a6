// neural_bandit.cu — NeuralBandit (a value network trained on the observed rewards) driven by PolicyLearner.learn or called
// directly on a caller's batch (PearlAgent.learn_batch / offline_learning), its scoring and its act with NoExploration,
// SquareCB or FastCB, replacing
//   policy_learners/contextual_bandits/neural_bandit.py                learn_batch (forward, weighted MSE / L1 loss,
//       AdamW(amsgrad) step), act, get_scores
//   neural_networks/common/value_networks.py                           VanillaValueNetwork: Linear+ReLU, Linear+ReLU, Linear
//   exploration_modules/contextual_bandits/squarecb_exploration.py     SquareCBExploration / FastCBExploration.act
//   exploration_modules/common/no_exploration.py                       the first maximum over the available actions
//
// Network: p = L3(L2(L1(x))), L1 = relu(x W1^T + b1), L2 = relu(. W2^T + b2), L3 = . W3^T + b3 with one output.  Flat
// parameters in torch's parameters() order: W1 b1 W2 b2 W3 b3 (ac_nets.cuh's Mlp2 with out = 1).
//
// Round (one fixed launch sequence, captured per (batch, buffer) into a CUDA graph and replayed):
//   k_cb_load      rows x (state, or state || represented action), label y, weight w       (ridge.cuh)
//   forward        three contractions (mlp2_forward)
//   k_nb_head      one CTA: per row l = (p - y)^2 or |p - y| and dl/dp = 2 (p - y) or sign(p - y) (torch's backward
//                  forms, sign 0 at 0); fixed-order sums of w and w l; loss = sum w l / sum w (no short circuit: a zero
//                  sum gives torch's inf / NaN); then the gradient rows dl/dp * (fp32(1 / sum w) * w), the order in which
//                  autograd evaluates the division, the product with w and the loss's backward
//   backward       mlp2_backward (four contractions and k_head_bwd)
//   k_adamw        AdamW(amsgrad) over every parameter
//   k_nb_bump      the round counter advances
// The learning rate reaches a captured round through the per-call block (k_adamw's decay factor and the per-round
// scalars), so a learning-rate change needs no new capture.  No float atomics and a fixed summation order everywhere:
// bit-reproducible run to run, graph or eager, and independent of how the rounds are split into calls.
//
// Scoring (prl_nb_scores, prl_nb_act) runs the network over the n x S feature rows (k_cb_feat of ridge.cuh) in chunks
// of the workspace's rows, writing the raw network output.  act then takes
//   kind 0  NoExploration: k_cb_argmax, the first maximum over the available actions of each state
//   kind 1  SquareCB, kind 2 FastCB, one state: k_nb_explore (below), with the A exponential draws E the caller made
//           where the reference's Categorical(p).sample() makes them
// No host synchronisation.
#include <math.h>

#include <new>

#include "ac_nets.cuh"
#include "common.cuh"
#include "ridge.cuh"
#include "rounds.cuh"

using namespace prl;

namespace {

constexpr int kHeadThreads = 256;
constexpr int kExploreThreads = 256;

// per-call block the captured round reads through
struct NbCall {
    const int32_t *slots;                                     // [rounds][B] (learn)
    float *out_pred, *out_label, *out_weight;                 // [rounds][B] (label, weight optional)
    float *out_loss;                                          // [rounds]
    // learn_batch: the caller's dense batch
    const float *d_state, *d_action, *d_reward, *d_weight;   // d_weight may be null: every weight is 1
    int d_action_ld;
    float decay;                                              // AdamW decoupled decay 1 - lr * weight_decay
};

// fixed-order sum of one value per thread over the CTA: a tree over shared memory, red[blockDim.x]
template <int NT>
__device__ __forceinline__ float nb_cta_sum(float v, float *red) {
    const int t = threadIdx.x;
    red[t] = v;
    __syncthreads();
#pragma unroll
    for (int o = NT / 2; o; o >>= 1) {
        if (t < o) red[t] = __fadd_rn(red[t], red[t + o]);
        __syncthreads();
    }
    const float s = red[0];
    __syncthreads();
    return s;
}

// first maximum over the CTA: every thread holds its own first maximum (v, i) of indices ascending; ties go to the
// smaller index, so the result is the first maximum of the whole vector
template <int NT>
__device__ __forceinline__ int nb_cta_argmax(float v, int i, float *rv, int *ri) {
    const int t = threadIdx.x;
    rv[t] = v; ri[t] = i;
    __syncthreads();
#pragma unroll
    for (int o = NT / 2; o; o >>= 1) {
        if (t < o) {
            const float ov = rv[t + o];
            const int oi = ri[t + o];
            if (ov > rv[t] || (ov == rv[t] && oi < ri[t])) { rv[t] = ov; ri[t] = oi; }
        }
        __syncthreads();
    }
    const int r = ri[0];
    __syncthreads();
    return r;
}

// the head of a round, one CTA (see the header)
__global__ void __launch_bounds__(kHeadThreads) k_nb_head(int B, int loss, const float *__restrict__ P, const float *__restrict__ Y,
                                                          const float *__restrict__ W, float *__restrict__ dP,
                                                          const NbCall *__restrict__ call, const int *__restrict__ round_idx) {
    __shared__ float red[kHeadThreads];
    const int t = threadIdx.x;
    const size_t o = (size_t)(*round_idx) * B;
    float sw = 0.f, swl = 0.f;
    for (int r = t; r < B; r += kHeadThreads) {
        const float p = P[r], y = Y[r], w = W[r];
        const float e = __fsub_rn(p, y);
        float l, g;
        if (loss == 0) {                       // mse_loss: (p - y)^2, backward 2 (p - y)
            l = __fmul_rn(e, e);
            g = __fmul_rn(2.f, e);
        } else {                               // l1_loss: |p - y|, backward sign(p - y) (0 at 0)
            l = fabsf(e);
            g = e > 0.f ? 1.f : (e < 0.f ? -1.f : 0.f);
        }
        call->out_pred[o + r] = p;
        if (call->out_label) call->out_label[o + r] = y;
        if (call->out_weight) call->out_weight[o + r] = w;
        dP[r] = g;
        sw = __fadd_rn(sw, w);
        swl = __fadd_rn(swl, __fmul_rn(l, w));
    }
    const float s = nb_cta_sum<kHeadThreads>(sw, red);
    const float sl = nb_cta_sum<kHeadThreads>(swl, red);
    if (t == 0) call->out_loss[*round_idx] = __fdiv_rn(sl, s);
    const float inv = __fdiv_rn(1.f, s);
    for (int r = t; r < B; r += kHeadThreads) dP[r] = __fmul_rn(dP[r], __fmul_rn(inv, W[r]));
}

__global__ void k_nb_bump(int *round_idx) { *round_idx += 1; }

// one state's unnormalised probability of action i (squarecb_exploration.py get_unnormalize_prob), fp32 in the
// reference's order: SquareCB 1 / (A + gamma gap); FastCB (max - lb) / (A (max - lb) + gamma gap), or 1 / A when max <= lb
__device__ __forceinline__ float nb_unnorm(float v, float mx, int kind, float fA, float gamma, float dd, bool uniform) {
    const float gap = __fsub_rn(mx, v);
    if (kind == 1) return __fdiv_rn(1.f, __fadd_rn(fA, __fmul_rn(gamma, gap)));
    if (uniform) return __fdiv_rn(1.f, fA);
    return __fdiv_rn(dd, __fadd_rn(__fmul_rn(fA, dd), __fmul_rn(gamma, gap)));
}

__device__ __forceinline__ float nb_clamp(float v, int clamp, float lb, float ub) {
    return clamp && !isnan(v) ? fminf(fmaxf(v, lb), ub) : v;
}

// SquareCB (kind 1) / FastCB (kind 2) act over one state's A values, one CTA: clamp, the first maximum, the unnormalised
// p with p[max] = 0 and then 1 - sum p, pn = p / sum p (Categorical's normalisation), and the sample as torch's one-sample
// multinomial takes it: the first maximum of pn / E over the caller's A exponential draws.  Sums in a fixed order (not
// torch's), so p may differ from the reference's in the last places.  Values are re-derived in every pass (the same
// arithmetic each time), so any A fits.  out_prob (optional) = pn.
__global__ void __launch_bounds__(kExploreThreads) k_nb_explore(int A, const float *__restrict__ values, int kind, float gamma, float lb,
                                                                float ub, int clamp, const float *__restrict__ E,
                                                                float *__restrict__ out_prob, int32_t *__restrict__ out_index) {
    __shared__ float rv[kExploreThreads];
    __shared__ int ri[kExploreThreads];
    const int t = threadIdx.x;
    float bv = -INFINITY;
    int bi = A;
    for (int i = t; i < A; i += kExploreThreads) {
        const float v = nb_clamp(values[i], clamp, lb, ub);
        if (bi == A || v > bv) { bv = v; bi = i; }
    }
    const int im = nb_cta_argmax<kExploreThreads>(bv, bi, rv, ri);
    const float mx = nb_clamp(values[im], clamp, lb, ub);
    const float fA = (float)A, dd = __fsub_rn(mx, lb);
    const bool uniform = kind == 2 && mx <= lb;
    float cs = 0.f;
    for (int i = t; i < A; i += kExploreThreads)
        if (i != im) cs = __fadd_rn(cs, nb_unnorm(nb_clamp(values[i], clamp, lb, ub), mx, kind, fA, gamma, dd, uniform));
    const float pmax = __fsub_rn(1.f, nb_cta_sum<kExploreThreads>(cs, rv));
    float s = 0.f;
    for (int i = t; i < A; i += kExploreThreads)
        s = __fadd_rn(s, i == im ? pmax : nb_unnorm(nb_clamp(values[i], clamp, lb, ub), mx, kind, fA, gamma, dd, uniform));
    const float tot = nb_cta_sum<kExploreThreads>(s, rv);
    bv = -INFINITY;
    bi = A;
    for (int i = t; i < A; i += kExploreThreads) {
        const float p = i == im ? pmax : nb_unnorm(nb_clamp(values[i], clamp, lb, ub), mx, kind, fA, gamma, dd, uniform);
        const float pn = __fdiv_rn(p, tot);
        if (out_prob) out_prob[i] = pn;
        const float q = __fdiv_rn(pn, E[i]);
        if (bi == A || q > bv) { bv = q; bi = i; }
    }
    const int ic = nb_cta_argmax<kExploreThreads>(bv, bi, rv, ri);
    if (t == 0) *out_index = ic < A ? ic : 0;
}

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_nb : Rounds<prl_nb, NbCall> {
    static constexpr const char *kFn = "prl_nb", *kName = "NeuralBandit";
    static constexpr int kGraphs = 2;    // buffer rounds and learn_batch
    prl_nb_cfg cfg;
    Mlp2 net;
    int f, rows;                     // network input width, rows of the row buffers (learn and scoring)
    float *w, *m, *v, *vmax;         // flat parameters and AdamW state [P]
    // workspace
    float *X, *H1, *H2, *P, *Y, *W, *dP, *dH2, *dH1, *g;
    void fill_call(NbCall &k) const { k.decay = (float)(1.0 - cfg.lr * cfg.weight_decay); }
    static int round(prl_nb *s, prl_buf *buf, int B, cudaStream_t st);
    void values(GemmLauncher &L, int n, const float *state, int n_space, const float *act_feat, float *out) const;
};

static int nb_check(const prl_nb_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim >= 0 && c->action_dim >= 0 && c->obs_dim + c->action_dim >= 1, "obs_dim + action_dim must be positive");
    PRL_REQUIRE(c->h1 >= 1 && c->h2 >= 1, "hidden_dims must be positive");
    PRL_REQUIRE(c->action_rep >= 0 && c->action_rep <= 2, "action_rep must be 0 (none), 1 (one-hot) or 2 (binary)");
    PRL_REQUIRE(c->action_rep != 1 || c->action_dim == c->n_actions, "a one-hot representation has action_dim = n_actions");
    PRL_REQUIRE(c->action_rep != 2 || (c->action_dim >= 1 && c->action_dim <= 30 && c->n_actions <= (1 << c->action_dim)),
                "a binary representation needs 1 <= action_dim <= 30 bits and n_actions <= 2^action_dim");
    PRL_REQUIRE(c->loss == 0 || c->loss == 1, "loss must be 0 (mse) or 1 (mae)");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0 && c->score_rows >= 0, "max_batch / max_rounds must be positive");
    const int64_t R = c->max_batch > c->score_rows ? c->max_batch : c->score_rows;
    const int64_t f = c->obs_dim + c->action_dim, wide = f > c->h1 ? (f > c->h2 ? f : c->h2) : (c->h1 > c->h2 ? c->h1 : c->h2);
    PRL_REQUIRE(R * wide < ((int64_t)1 << 31), "max(max_batch, score_rows) * the widest layer must stay below 2^31 (32-bit element offsets)");
    PRL_REQUIRE((int64_t)c->h1 * f + (int64_t)c->h2 * c->h1 + c->h1 + 2 * (int64_t)c->h2 + 1 < ((int64_t)1 << 31),
                "the parameter count must stay below 2^31");
    return PRL_OK;
}

static void nb_layout(prl_nb *s) {
    const prl_nb_cfg &c = s->cfg;
    s->f = c.obs_dim + c.action_dim;
    s->net = mlp2(s->f, c.h1, c.h2, 1);
    s->rows = c.max_batch > c.score_rows ? c.max_batch : c.score_rows;
}

// the workspace, in order; base == null: only its size
static int64_t nb_carve(prl_nb *s, void *base) {
    const prl_nb_cfg &c = s->cfg;
    const int64_t R = s->rows, B = c.max_batch, F = s->f, H1 = c.h1, H2 = c.h2;
    Carve w{(char *)base};
    w(s->X, R * F); w(s->H1, R * H1); w(s->H2, R * H2); w(s->P, R);
    w(s->Y, B); w(s->W, B); w(s->dP, B); w(s->dH2, B * H2); w(s->dH1, B * H1);
    w(s->g, (int64_t)s->net.P);
    s->carve_tail(w, c.max_rounds, B);
    return w.bytes;
}

extern "C" int64_t prl_nb_param_count(const prl_nb_cfg *c) {
    if (nb_check(c)) return -1;
    prl_nb t; t.cfg = *c; nb_layout(&t);
    return t.net.P;
}

extern "C" int64_t prl_nb_workspace_bytes(const prl_nb_cfg *c) {
    if (nb_check(c)) return -1;
    prl_nb t; t.cfg = *c; nb_layout(&t);
    return nb_carve(&t, nullptr);
}

extern "C" int prl_nb_create(prl_nb **out, const prl_nb_cfg *cfg, float *w, float *m, float *v, float *vmax, int64_t adam_step,
                             void *workspace) {
    PRL_REQUIRE(out && w && m && v && vmax && workspace, "null argument");
    int rc = nb_check(cfg);
    if (rc) return rc;
    PRL_REQUIRE(adam_step >= 0, "the AdamW step count must be non-negative");
    prl_nb *s = new (std::nothrow) prl_nb();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    nb_layout(s);
    s->w = w; s->m = m; s->v = v; s->vmax = vmax;
    s->adam_step = adam_step;
    nb_carve(s, workspace);
    return prl_nb::open(s, out);
}
extern "C" int prl_nb_destroy(prl_nb *s) { return prl_nb::destroy(s); }
extern "C" int prl_nb_set_graph(prl_nb *s, int enable) { return prl_nb::set_graph(s, enable); }
extern "C" int prl_nb_set_lr(prl_nb *s, double lr) { return prl_nb::set_lr(s, lr); }
extern "C" int64_t prl_nb_adam_step(const prl_nb *s) { return prl_nb::adam_step_of(s); }
extern "C" int prl_nb_set_adam_step(prl_nb *s, int64_t step) { return prl_nb::set_adam_step(s, step); }
extern "C" int64_t prl_nb_last_launches(const prl_nb *s) { return prl_nb::last_launches_of(s); }
extern "C" int64_t prl_nb_graph_captures(const prl_nb *s) { return s ? s->graphs.captures : -1; }

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
int prl_nb::round(prl_nb *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_nb_cfg &c = s->cfg;
    const Mlp2 &n = s->net;
    const int eb = 256;
    GemmLauncher L; L.st = st;
    k_cb_load<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf ? buf->records : nullptr, buf ? buf->lay : prl_buf_layout{}, c.obs_dim,
                                                    c.action_dim, c.action_rep, s->call, s->round_idx, B, s->X, s->Y, s->W);
    mlp2_forward(L, n, s->w, s->X, B, s->H1, s->H2, s->P);
    k_nb_head<<<1, kHeadThreads, 0, st>>>(B, c.loss, s->P, s->Y, s->W, s->dP, s->call, s->round_idx);
    mlp2_backward(L, n, s->w, s->g, s->dP, s->X, s->H1, s->H2, s->dH2, s->dH1, B);   // + one k_head_bwd
    const AdamHp hp = adam_hp(0.0, c.beta1, c.beta2, c.eps, c.weight_decay);         // decay: call->decay
    k_adamw<<<(n.P + eb - 1) / eb, eb, 0, st>>>(n.P, s->w, s->m, s->v, s->vmax, s->g, hp, s->scal, s->round_idx, nullptr, 0.f, 0.f,
                                               &s->call->decay);
    k_nb_bump<<<1, 1, 0, st>>>(s->round_idx);
    s->launches_per_round = L.count + 5;   // load, head, k_head_bwd, AdamW, bump
    return PRL_OK;
}

extern "C" int prl_nb_learn(prl_nb *s, prl_buf *buf, int rounds, int batch, float *out_pred, float *out_label, float *out_weight,
                            float *out_loss, int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && out_pred && out_loss, "null argument");
    PRL_REQUIRE(s->cfg.action_rep != 0 || s->cfg.action_dim == 0,
                "learn over a buffer needs the state alone (action_dim 0) or a one-hot or binary action representation");
    NbCall call{};
    call.out_pred = out_pred; call.out_label = out_label; call.out_weight = out_weight; call.out_loss = out_loss;
    return prl_nb::learn(s, buf, rounds, batch, 0, out_logical, call, stream_);
}

extern "C" int prl_nb_learn_batch(prl_nb *s, int batch, const float *state, const float *action, const float *reward,
                                  const float *weight, float *out_pred, float *out_loss, void *stream_) {
    PRL_REQUIRE(s && (state || s->cfg.obs_dim == 0) && (action || s->cfg.action_dim == 0) && reward && out_pred && out_loss,
                "null argument");
    NbCall dense{};
    dense.d_state = state; dense.d_action = action; dense.d_reward = reward; dense.d_weight = weight;
    dense.d_action_ld = s->cfg.action_dim;
    dense.out_pred = out_pred; dense.out_loss = out_loss;
    return prl_nb::learn_batch(s, batch, 0, dense, stream_);
}

// the network's output over the n x n_space feature rows into out, in chunks of the workspace's rows
void prl_nb::values(GemmLauncher &L, int n, const float *state, int n_space, const float *act_feat, float *out) const {
    const long long total = (long long)n * n_space;
    for (long long r0 = 0; r0 < total; r0 += rows) {
        const int mr = (int)(total - r0 < rows ? total - r0 : rows);
        k_cb_feat<<<(mr * 32 + 255) / 256, 256, 0, L.st>>>(mr, r0, n_space, cfg.obs_dim, cfg.action_dim, state, act_feat, X);
        mlp2_forward(L, net, w, X, mr, H1, H2, out + r0);
    }
}

static int nb_scores_check(const prl_nb *s, int n, const float *state, int n_space, const float *act_feat, const float *out) {
    PRL_REQUIRE(s && out && (state || s->cfg.obs_dim == 0) && (act_feat || s->cfg.action_dim == 0), "null argument");
    PRL_REQUIRE(n >= 0 && n_space >= 1 && (int64_t)n * n_space < ((int64_t)1 << 31), "n * n_space must be in [0, 2^31)");
    return PRL_OK;
}

extern "C" int prl_nb_scores(prl_nb *s, int n, const float *state, int n_space, const float *act_feat, float *out_scores, void *stream_) {
    int rc = nb_scores_check(s, n, state, n_space, act_feat, out_scores);
    if (rc) return rc;
    if (n == 0) return PRL_OK;
    GemmLauncher L; L.st = (cudaStream_t)stream_;
    s->values(L, n, state, n_space, act_feat, out_scores);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

extern "C" int prl_nb_explore(int n_space, const float *values, int kind, double gamma, double lb, double ub, int clamp, const float *E,
                              float *out_prob, int32_t *out_index, void *stream_) {
    PRL_REQUIRE(values && E && out_index, "null argument");
    PRL_REQUIRE(n_space >= 1, "n_space must be positive");
    PRL_REQUIRE(kind == 1 || kind == 2, "kind must be 1 (SquareCB) or 2 (FastCB)");
    k_nb_explore<<<1, kExploreThreads, 0, (cudaStream_t)stream_>>>(n_space, values, kind, (float)gamma, (float)lb, (float)ub,
                                                                   kind == 2 ? 1 : (clamp != 0), E, out_prob, out_index);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

extern "C" int prl_nb_act(prl_nb *s, int n, const float *state, int n_space, const float *act_feat, int kind, double gamma, double lb,
                          double ub, int clamp, const float *E, const uint8_t *mask, float *out_values, float *out_prob,
                          int32_t *out_index, void *stream_) {
    int rc = nb_scores_check(s, n, state, n_space, act_feat, out_values);
    if (rc) return rc;
    PRL_REQUIRE(out_index, "null argument");
    PRL_REQUIRE(kind >= 0 && kind <= 2, "kind must be 0 (NoExploration), 1 (SquareCB) or 2 (FastCB)");
    PRL_REQUIRE(kind == 0 || n == 1, "SquareCB / FastCB act over one state at a time (n = %d)", n);
    PRL_REQUIRE(kind == 0 || E, "SquareCB / FastCB need the exponential draws E");
    if (n == 0) return PRL_OK;
    cudaStream_t st = (cudaStream_t)stream_;
    GemmLauncher L; L.st = st;
    s->values(L, n, state, n_space, act_feat, out_values);
    if (kind == 0) {
        k_cb_argmax<<<(n + 255) / 256, 256, 0, st>>>(n, n_space, out_values, mask, out_index);
        PRL_CUDA(cudaGetLastError());
        return PRL_OK;
    }
    return prl_nb_explore(n_space, out_values, kind, gamma, lb, ub, clamp, E, out_prob, out_index, stream_);
}
