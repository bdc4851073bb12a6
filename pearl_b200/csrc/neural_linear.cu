// neural_linear.cu — NeuralLinearBandit (neural LinUCB) driven by PolicyLearner.learn or called directly on a caller's
// batch (PearlAgent.learn_batch / offline_learning), and its UCB scoring, replacing
//   policy_learners/contextual_bandits/neural_linear_bandit.py      learn_batch (forward, weighted loss, AdamW(amsgrad) step,
//       the ridge on the pre-step nn_output, _maybe_apply_discounting), act / get_scores
//   neural_networks/contextual_bandit/neural_linear_regression.py   forward_with_intermediate_values (mu from
//       linear_layer_e2e, or from the ridge's coefs), calculate_sigma
//   neural_networks/common/utils.py                                  mlp_block with two hidden layers, ReLU, and
//   neural_networks/common/residual_wrapper.py                       x + layer(x) on every layer of equal in / out width
//
// Network: nn_output = L3(L2(L1(x))), L1 = relu(x W1^T + b1), L2 = relu(. W2^T + b2), L3 = . W3^T + b3 (h2 -> h2, no
// activation), each wrapped as x + L(x) when use_skip_connections and its widths agree (L3 always then).  Flat parameters
// in torch's parameters() order: W1 b1 W2 b2 W3 b3 (ac_nets.cuh's Mlp2 with out = h2), then linear_layer_e2e.weight [h2].
//
// Round (one fixed launch sequence, captured per (batch, buffer, variant) into a CUDA graph and replayed):
//   k_cb_load      rows x (state, or state || represented action), label y, weight w       (ridge.cuh)
//   forward        three contractions; k_nl_add for each residual
//   k_nl_rows      per row: mu = nn_output . e2e weight, or [1, nn_output] . coefs (the coefs before this round's ridge
//                  update); p = activation(mu); l = mse / l1 / bce(p, y); dl/dmu as torch's backward forms evaluate it
//   k_nl_loss      one CTA, fixed order: sum w, sum w l, sum p -> loss (0 when sum w = 0) and mu_scores of the round
//   k_nl_grad      dL/dnn_output[b][j] = dl/dmu_b * (w_b / sum w) * v[j], v = e2e weight or coefs[1:] (constants)
//   backward       the MLP's parameter gradient (ac_nets.cuh's mlp2_backward, or the residual chain), and the e2e weight
//                  gradient as one more contraction (e2e only)
//   k_adamw        AdamW(amsgrad) over P_mlp + h2 parameters (e2e), or P_mlp: without e2e linear_layer_e2e never gets a
//                  gradient, so torch's AdamW skips it (no state, no weight decay)
//   k_cb_stats, k_cb_reduce, k_cb_solve   the ridge on the nn_output of the forward pass above (ridge.cuh)
// Variant 1 (a learn_batch whose weights sum to 0, decided on the host as the reference's `.item()` does) drops k_nl_grad,
// the backward and AdamW: the reference takes no optimizer step, and the AdamW step count does not advance.  The ridge
// is still updated and re-solved.
// The learning rate reaches a captured round through the per-call block (the AdamW scalars and the decay factor), so a
// learning-rate change needs no new capture.  No float atomics and a fixed summation order everywhere: bit-reproducible
// run to run, graph or eager, and independent of how the rounds are split into calls.
//
// Scoring (prl_nlb_scores) runs the network over the n x S feature rows in chunks of the workspace's rows, then per row
// mu (as above) and sigma = sqrt([1, nn_output]^T inv_A [1, nn_output]) (NaN -> 0), combined as act or get_scores do;
// the argmax of ridge.cuh follows.  No host synchronisation.  Thompson sampling (prl_nlb_ts_scores) runs the same network
// pass, then [1, nn_output] . theta with theta from ridge.cuh's k_cb_ts_sample.
#include <math.h>

#include <new>

#include "ac_nets.cuh"
#include "common.cuh"
#include "ridge.cuh"
#include "rounds.cuh"

using namespace prl;

namespace {

constexpr int kMaxH2 = kMaxD - 1;   // the ridge's width: d = h2 + 1 <= 128

// per-call block the captured round reads through
struct NlCall {
    const int32_t *slots;                                     // [rounds][B] (learn)
    float *out_pred, *out_label, *out_weight;                 // [rounds][B] (label, weight optional)
    float *out_loss, *out_mu;                                 // [rounds]
    // learn_batch: the caller's dense batch
    const float *d_state, *d_action, *d_reward, *d_weight;   // d_weight may be null: every weight is 1
    int d_action_ld;
    float decay;                                              // AdamW decoupled decay 1 - lr * weight_decay
};

// the head's settings
struct NlHead {
    int h2, e2e, loss, sigmoid;   // loss 0: mse, 1: mae (l1), 2: binary cross-entropy
};

// y[i] = a[i] + b[i]: a residual connection, x + layer(x)
__global__ void k_nl_add(int n, const float *__restrict__ a, const float *__restrict__ b, float *__restrict__ y) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < (unsigned)n) y[i] = __fadd_rn(a[i], b[i]);
}

// backward of a layer whose input feeds a ReLU layer below: o = u + res (res: the gradient the residual passes through,
// may be null), in place; z = o where the inner activation a > 0, else 0 (torch masks by the ReLU's own output)
__global__ void k_nl_res_bwd(int n, float *__restrict__ u, const float *__restrict__ res, const float *__restrict__ a,
                             float *__restrict__ z) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (unsigned)n) return;
    const float o = res ? __fadd_rn(u[i], res[i]) : u[i];
    u[i] = o;
    z[i] = a[i] > 0.f ? o : 0.f;
}

__device__ __forceinline__ float nl_mu(const float *__restrict__ x, const float *__restrict__ we, const float *__restrict__ coefs,
                                       const NlHead &h, int lane) {
    float s = 0.f;
    if (h.e2e)
        for (int j = lane; j < h.h2; j += 32) s = fmaf(x[j], we[j], s);
    else
        for (int j = lane; j < h.h2; j += 32) s = fmaf(x[j], coefs[j + 1], s);
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return h.e2e ? s : __fadd_rn(coefs[0], s);
}

// one warp per row: mu, p = activation(mu), the per-row loss times its weight (WL), dl/dmu (G, without the weight), the
// report of the round
__global__ void __launch_bounds__(256) k_nl_rows(int B, NlHead h, const float *__restrict__ N, const float *__restrict__ we,
                                                 const float *__restrict__ coefs, const float *__restrict__ Y,
                                                 const float *__restrict__ W, float *__restrict__ Pr, float *__restrict__ WL,
                                                 float *__restrict__ G, const NlCall *__restrict__ call,
                                                 const int *__restrict__ round_idx) {
    const int lane = threadIdx.x & 31;
    const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (r >= B) return;
    const float mu = nl_mu(N + (size_t)r * h.h2, we, coefs, h, lane);
    if (lane) return;
    const float y = Y[r], w = W[r];
    const float p = h.sigmoid ? 1.f / (1.f + expf(-mu)) : mu;
    const float e = p - y;
    float l, g;
    if (h.loss == 0) {                         // mse_loss: (p - y)^2, backward 2 (p - y)
        l = e * e;
        g = 2.f * e;
    } else if (h.loss == 1) {                  // l1_loss: |p - y|, backward sign(p - y) (0 at 0)
        l = fabsf(e);
        g = e > 0.f ? 1.f : (e < 0.f ? -1.f : 0.f);
    } else {                                   // binary_cross_entropy: logs clamped at -100, backward (p - y) / max(p (1 - p), 1e-12)
        const float lp = fmaxf(logf(p), -100.f), l1p = fmaxf(logf(1.f - p), -100.f);
        l = -(y * lp + (1.f - y) * l1p);
        g = e / fmaxf(p * (1.f - p), 1e-12f);
    }
    if (h.sigmoid) g = g * (1.f - p) * p;      // sigmoid backward: grad (1 - p) p
    const size_t o = (size_t)(*round_idx) * B + r;
    call->out_pred[o] = p;
    if (call->out_label) call->out_label[o] = y;
    if (call->out_weight) call->out_weight[o] = w;
    Pr[r] = p;
    WL[r] = __fmul_rn(l, w);
    G[r] = g;
}

// one CTA: sum w, sum w l and sum p in a fixed order (per-thread strided sums, then a tree); sw[0] = sum w for k_nl_grad;
// the round's loss (sum w l / sum w, 0 when sum w = 0, as the reference's short circuit) and mu_scores (mean p)
__global__ void __launch_bounds__(1024) k_nl_loss(int B, const float *__restrict__ W, const float *__restrict__ WL,
                                                  const float *__restrict__ Pr, float *__restrict__ sw,
                                                  const NlCall *__restrict__ call, const int *__restrict__ round_idx) {
    __shared__ float rw[1024], rl[1024], rp[1024];
    const int t = threadIdx.x;
    float a = 0.f, b = 0.f, c = 0.f;
    for (int r = t; r < B; r += 1024) {
        a = __fadd_rn(a, W[r]);
        b = __fadd_rn(b, WL[r]);
        c = __fadd_rn(c, Pr[r]);
    }
    rw[t] = a; rl[t] = b; rp[t] = c;
    __syncthreads();
    for (int o = 512; o; o >>= 1) {
        if (t < o) {
            rw[t] = __fadd_rn(rw[t], rw[t + o]);
            rl[t] = __fadd_rn(rl[t], rl[t + o]);
            rp[t] = __fadd_rn(rp[t], rp[t + o]);
        }
        __syncthreads();
    }
    if (t == 0) {
        const float s = rw[0];
        sw[0] = s;
        call->out_loss[*round_idx] = s == 0.f ? 0.f : __fdiv_rn(rl[0], s);
        call->out_mu[*round_idx] = __fdiv_rn(rp[0], (float)B);
    }
}

// dL/dnn_output[b][j] = gm_b v[j], gm_b = dl/dmu_b * (w_b / sum w) (also written to GM for the e2e weight gradient);
// v = the e2e weight, or coefs[1:] held constant
__global__ void k_nl_grad(int B, NlHead h, const float *__restrict__ G, const float *__restrict__ W, const float *__restrict__ sw,
                          const float *__restrict__ we, const float *__restrict__ coefs, float *__restrict__ GM,
                          float *__restrict__ dN) {
    const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (unsigned)(B * h.h2)) return;
    const int e = (int)t, b = e / h.h2, j = e - b * h.h2;
    const float gm = __fmul_rn(G[b], __fdiv_rn(W[b], sw[0]));
    if (j == 0) GM[b] = gm;
    dN[e] = __fmul_rn(gm, h.e2e ? we[j] : coefs[j + 1]);
}

// scores of rows [r0, r0 + m), one warp per row x1 = [1, nn_output]: mu as k_nl_rows, sigma = sqrt(x1^T inv_A x1) (NaN -> 0)
//   mode 0 (act):                            mu + alpha sigma
//   mode 1 (get_scores, combined):           activation(mu + alpha sigma)
//   mode 2 (get_scores, separate_uncertainty): activation(mu) + alpha sigma
__global__ void __launch_bounds__(256) k_nl_scores(int m, long long r0, NlHead h, const float *__restrict__ N,
                                                   const float *__restrict__ we, const float *__restrict__ inv_A,
                                                   const float *__restrict__ coefs, int mode, float alpha,
                                                   float *__restrict__ out) {
    __shared__ float xs[8][kMaxD];
    const int lane = threadIdx.x & 31, wb = threadIdx.x >> 5, w = blockIdx.x * 8 + wb;
    if (w >= m) return;
    const int d = h.h2 + 1;
    const float *n = N + (size_t)w * h.h2;
    float *x = xs[wb];
    for (int c = lane; c < d; c += 32) x[c] = c == 0 ? 1.f : n[c - 1];
    __syncwarp();
    const float mu = nl_mu(n, we, coefs, h, lane);
    float q = 0.f;
    for (int j = lane; j < d; j += 32) {
        float t = 0.f;
        for (int i = 0; i < d; i++) t = fmaf(x[i], inv_A[(size_t)i * d + j], t);
        q = fmaf(t, x[j], q);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    if (lane) return;
    float sg = sqrtf(q);
    if (isnan(sg)) sg = 0.f;
    const float u = __fmul_rn(alpha, sg);
    float v;
    if (mode == 0) v = __fadd_rn(mu, u);
    else if (mode == 1) { v = __fadd_rn(mu, u); if (h.sigmoid) v = 1.f / (1.f + expf(-v)); }
    else v = __fadd_rn(h.sigmoid ? 1.f / (1.f + expf(-mu)) : mu, u);
    out[r0 + w] = v;
}

// Thompson sampling scores of rows [r0, r0 + m), one warp per row: [1, nn_output] . theta (the sampled coefficients, in
// place of the ridge's coefs whatever e2e is), then the output activation when `activate` (get_scores without
// separate_uncertainty); act and separate_uncertainty's get_scores take the product as it is
__global__ void __launch_bounds__(256) k_nl_ts_scores(int m, long long r0, NlHead h, const float *__restrict__ N,
                                                      const float *__restrict__ theta, int activate, float *__restrict__ out) {
    const int lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= m) return;
    h.e2e = 0;
    const float mu = nl_mu(N + (size_t)w * h.h2, nullptr, theta, h, lane);
    if (lane) return;
    out[r0 + w] = activate && h.sigmoid ? 1.f / (1.f + expf(-mu)) : mu;
}

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_nlb : Rounds<prl_nlb, NlCall> {
    static constexpr const char *kFn = "prl_nlb", *kName = "NeuralLinearBandit";
    static constexpr int kGraphs = 3;    // buffer rounds, learn_batch, and learn_batch's zero-weight variant
    prl_nlb_cfg cfg;
    Mlp2 net;
    int f, d, rows;                  // network input width, ridge width + 1, rows of the row buffers (learn and scoring)
    bool r1, r2, r3;                 // residual connections of layers 1, 2, 3
    int zero_weight = 0;             // the next learn_batch runs variant 1
    float *w, *m, *v, *vmax;         // flat parameters and AdamW state [P_mlp + h2]
    float *A, *b, *sum_weight, *inv_A, *coefs;
    double *last_discount;
    // workspace
    float *X, *A1, *H1, *A2, *H2, *T3, *N, *Y, *W, *Pr, *WL, *G, *GM, *sw, *dN, *U2, *Z2, *U1, *Z1, *g, *gdb, *P;
    NlHead head() const { return NlHead{cfg.h2, cfg.e2e, cfg.loss, cfg.sigmoid}; }
    int n_opt() const { return net.P + (cfg.e2e ? cfg.h2 : 0); }
    void fill_call(NlCall &k) const { k.decay = (float)(1.0 - cfg.lr * cfg.weight_decay); }
    int buffer_ok(const prl_buf *buf) const {
        PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.obs_dim == cfg.obs_dim && buf->desc.n_actions == cfg.n_actions,
                    "NeuralLinearBandit needs a discrete-action buffer with obs_dim = %d and n_actions = %d", cfg.obs_dim, cfg.n_actions);
        PRL_REQUIRE(buf->shard_world <= 1, "the buffer is one shard of a multi-GPU buffer: NeuralLinearBandit samples local buffers only");
        return PRL_OK;
    }
    int variant(int) const { return zero_weight; }
    int round_variant(prl_buf *buf, int B, int v, cudaStream_t st);
    void forward(GemmLauncher &L, int rows_) const;
    static int round(prl_nlb *s, prl_buf *buf, int B, cudaStream_t st) { return s->round_variant(buf, B, 0, st); }
};

static int nl_check(const prl_nlb_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim >= 0 && c->action_dim >= 0 && c->obs_dim + c->action_dim >= 1, "obs_dim + action_dim must be positive");
    PRL_REQUIRE(c->h1 >= 1, "hidden_dims[0] must be positive");
    PRL_REQUIRE(c->h2 >= 1 && c->h2 <= kMaxH2, "hidden_dims[-1] = %d: the ridge solve supports 1 to %d features (%d with the intercept)",
                c->h2, kMaxH2, kMaxD);
    PRL_REQUIRE(c->action_rep >= 0 && c->action_rep <= 2, "action_rep must be 0 (none), 1 (one-hot) or 2 (binary)");
    PRL_REQUIRE(c->action_rep != 1 || c->action_dim == c->n_actions, "a one-hot representation has action_dim = n_actions");
    PRL_REQUIRE(c->action_rep != 2 || (c->action_dim >= 1 && c->action_dim <= 30 && c->n_actions <= (1 << c->action_dim)),
                "a binary representation needs 1 <= action_dim <= 30 bits and n_actions <= 2^action_dim");
    PRL_REQUIRE(c->loss >= 0 && c->loss <= 2, "loss must be 0 (mse), 1 (mae) or 2 (cross entropy)");
    PRL_REQUIRE(c->loss != 2 || c->sigmoid, "the cross-entropy loss needs the sigmoid output activation");
    PRL_REQUIRE(c->l2_reg_lambda > 0.0, "l2_reg_lambda must be positive (A + lambda I must be invertible)");
    PRL_REQUIRE(c->gamma > 0.0 && c->gamma <= 1.0, "gamma must be in (0, 1]");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0 && c->score_rows >= 0, "max_batch / max_rounds must be positive");
    const int64_t R = c->max_batch > c->score_rows ? c->max_batch : c->score_rows;
    const int64_t f = c->obs_dim + c->action_dim, wide = f > c->h1 ? (f > c->h2 ? f : c->h2) : (c->h1 > c->h2 ? c->h1 : c->h2);
    PRL_REQUIRE(R * wide < ((int64_t)1 << 31), "max(max_batch, score_rows) * the widest layer must stay below 2^31 (32-bit element offsets)");
    PRL_REQUIRE((int64_t)c->h1 * f + (int64_t)c->h2 * c->h1 + (int64_t)c->h2 * c->h2 + c->h1 + 3 * (int64_t)c->h2 < ((int64_t)1 << 31),
                "the parameter count must stay below 2^31");
    return PRL_OK;
}

static void nl_layout(prl_nlb *s) {
    const prl_nlb_cfg &c = s->cfg;
    s->f = c.obs_dim + c.action_dim;
    s->d = c.h2 + 1;
    s->net = mlp2(s->f, c.h1, c.h2, c.h2);
    s->rows = c.max_batch > c.score_rows ? c.max_batch : c.score_rows;
    s->r1 = c.skip && s->f == c.h1;
    s->r2 = c.skip && c.h1 == c.h2;
    s->r3 = c.skip != 0;
}

// the workspace, in order; base == null: only its size
static int64_t nl_carve(prl_nlb *s, void *base) {
    const prl_nlb_cfg &c = s->cfg;
    const int64_t R = s->rows, B = c.max_batch, F = s->f, H1 = c.h1, H2 = c.h2, chunks = (B + kChunk - 1) / kChunk;
    Carve w{(char *)base};
    w(s->X, R * F); w(s->A1, R * H1); w(s->A2, R * H2); w(s->T3, R * H2);
    // the residual outputs, or aliases of the inner ones
    if (s->r1) w(s->H1, R * H1); else s->H1 = s->A1;
    if (s->r2) w(s->H2, R * H2); else s->H2 = s->A2;
    if (s->r3) w(s->N, R * H2); else s->N = s->T3;
    w(s->Y, B); w(s->W, B); w(s->Pr, B); w(s->WL, B); w(s->G, B); w(s->GM, B); w(s->sw, 64);
    w(s->dN, B * H2); w(s->U2, B * H2); w(s->Z2, B * H2); w(s->U1, B * H1); w(s->Z1, B * H1);
    w(s->g, (int64_t)s->net.P + H2); w(s->gdb, 64);
    w(s->P, chunks * cb_entries(s->d));
    s->carve_tail(w, c.max_rounds, B);
    return w.bytes;
}

extern "C" int64_t prl_nlb_param_count(const prl_nlb_cfg *c) {
    if (nl_check(c)) return -1;
    prl_nlb t; t.cfg = *c; nl_layout(&t);
    return t.net.P + c->h2;
}

extern "C" int64_t prl_nlb_workspace_bytes(const prl_nlb_cfg *c) {
    if (nl_check(c)) return -1;
    prl_nlb t; t.cfg = *c; nl_layout(&t);
    return nl_carve(&t, nullptr);
}

extern "C" int prl_nlb_create(prl_nlb **out, const prl_nlb_cfg *cfg, float *w, float *m, float *v, float *vmax, int64_t adam_step,
                              float *A, float *b, float *sum_weight, float *inv_A, float *coefs, double *last_discount, void *workspace) {
    PRL_REQUIRE(out && w && m && v && vmax && A && b && sum_weight && inv_A && coefs && last_discount && workspace, "null argument");
    int rc = nl_check(cfg);
    if (rc) return rc;
    PRL_REQUIRE(adam_step >= 0, "the AdamW step count must be non-negative");
    PRL_CUDA(cb_solve_prepare());
    prl_nlb *s = new (std::nothrow) prl_nlb();
    if (!s) return fail(PRL_ENOMEM, "out of host memory");
    s->cfg = *cfg;
    nl_layout(s);
    s->w = w; s->m = m; s->v = v; s->vmax = vmax;
    s->A = A; s->b = b; s->sum_weight = sum_weight; s->inv_A = inv_A; s->coefs = coefs; s->last_discount = last_discount;
    s->adam_step = adam_step;
    nl_carve(s, workspace);
    return prl_nlb::open(s, out);
}
extern "C" int prl_nlb_destroy(prl_nlb *s) { return prl_nlb::destroy(s); }
extern "C" int prl_nlb_set_graph(prl_nlb *s, int enable) { return prl_nlb::set_graph(s, enable); }
extern "C" int prl_nlb_set_lr(prl_nlb *s, double lr) { return prl_nlb::set_lr(s, lr); }
extern "C" int64_t prl_nlb_adam_step(const prl_nlb *s) { return prl_nlb::adam_step_of(s); }
extern "C" int prl_nlb_set_adam_step(prl_nlb *s, int64_t step) { return prl_nlb::set_adam_step(s, step); }
extern "C" int64_t prl_nlb_last_launches(const prl_nlb *s) { return prl_nlb::last_launches_of(s); }
extern "C" int64_t prl_nlb_graph_captures(const prl_nlb *s) { return s ? s->graphs.captures : -1; }

// the network over rows_ rows of X: A1, H1, A2, H2, T3 and nn_output N
void prl_nlb::forward(GemmLauncher &L, int rows_) const {
    const Mlp2 &n = net;
    const int eb = 256;
    if (!r1 && !r2 && !r3) {
        mlp2_forward(L, n, w, X, rows_, A1, A2, T3);
        return;
    }
    L.fwd(mat(X, n.in), rows_, w + n.W1, n.in, 0, w + n.b1, 0, n.h1, n.in, true, A1, n.h1, 0);
    if (r1) { k_nl_add<<<(rows_ * n.h1 + eb - 1) / eb, eb, 0, L.st>>>(rows_ * n.h1, X, A1, H1); L.count++; }
    L.fwd(mat(H1, n.h1), rows_, w + n.W2, n.h1, 0, w + n.b2, 0, n.h2, n.h1, true, A2, n.h2, 0);
    if (r2) { k_nl_add<<<(rows_ * n.h2 + eb - 1) / eb, eb, 0, L.st>>>(rows_ * n.h2, H1, A2, H2); L.count++; }
    L.fwd(mat(H2, n.h2), rows_, w + n.W3, n.h2, 0, w + n.b3, 0, n.out, n.h2, false, T3, n.out, 0);
    if (r3) { k_nl_add<<<(rows_ * n.h2 + eb - 1) / eb, eb, 0, L.st>>>(rows_ * n.h2, H2, T3, N); L.count++; }
}

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
int prl_nlb::round_variant(prl_buf *buf, int B, int variant, cudaStream_t st) {
    const prl_nlb_cfg &c = cfg;
    const Mlp2 &n = net;
    const NlHead h = head();
    const int E = cb_entries(d), chunks = (B + kChunk - 1) / kChunk, eb = 256;
    GemmLauncher L; L.st = st;
    k_cb_load<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(buf ? buf->records : nullptr, buf ? buf->lay : prl_buf_layout{}, c.obs_dim,
                                                    c.action_dim, c.action_rep, call, round_idx, B, X, Y, W);
    forward(L, B);
    k_nl_rows<<<(B * 32 + eb - 1) / eb, eb, 0, st>>>(B, h, N, w + n.P, coefs, Y, W, Pr, WL, G, call, round_idx);
    k_nl_loss<<<1, 1024, 0, st>>>(B, W, WL, Pr, sw, call, round_idx);
    int extra = 3;
    if (variant == 0) {
        k_nl_grad<<<(B * c.h2 + eb - 1) / eb, eb, 0, st>>>(B, h, G, W, sw, w + n.P, coefs, GM, dN);
        if (!r1 && !r2 && !r3) {
            mlp2_backward(L, n, w, g, dN, X, A1, A2, U2, U1, B);
        } else {
            // layer 3: no activation, so its pre-activation gradient is dN itself
            L.bwd_w(dN, n.h2, 0, B, n.h2, mat(H2, n.h2), n.h2, g + n.W3, n.h2, 0, g + n.b3, 0);
            L.bwd_x(dN, n.h2, 0, B, n.h2, w + n.W3, n.h2, 0, 0, n.h2, U2, n.h2, 0, nullptr, 0, 0, false);
            k_nl_res_bwd<<<(B * n.h2 + eb - 1) / eb, eb, 0, st>>>(B * n.h2, U2, r3 ? dN : nullptr, A2, Z2);
            L.bwd_w(Z2, n.h2, 0, B, n.h2, mat(H1, n.h1), n.h1, g + n.W2, n.h1, 0, g + n.b2, 0);
            L.bwd_x(Z2, n.h2, 0, B, n.h2, w + n.W2, n.h1, 0, 0, n.h1, U1, n.h1, 0, nullptr, 0, 0, false);
            k_nl_res_bwd<<<(B * n.h1 + eb - 1) / eb, eb, 0, st>>>(B * n.h1, U1, r2 ? U2 : nullptr, A1, Z1);
            L.bwd_w(Z1, n.h1, 0, B, n.h1, mat(X, n.in), n.in, g + n.W1, n.in, 0, g + n.b1, 0);
            extra += 2;
        }
        if (c.e2e) L.bwd_w(GM, 1, 0, B, 1, mat(N, n.h2), n.h2, g + n.P, n.h2, 0, gdb, 0);
        const AdamHp hp = adam_hp(0.0, c.beta1, c.beta2, c.eps, c.weight_decay);   // decay: call->decay
        const int P = n_opt();
        k_adamw<<<(P + eb - 1) / eb, eb, 0, st>>>(P, w, m, v, vmax, g, hp, scal, round_idx, nullptr, 0.f, 0.f, &call->decay);
        extra += 2;
        if (!r1 && !r2 && !r3 && n.out == 1) extra += 1;   // mlp2_backward's k_head_bwd
    }
    k_cb_stats<<<dim3(chunks, (E + 255) / 256), 256, 0, st>>>(B, c.h2, N, Y, W, P);
    k_cb_reduce<<<(E + eb - 1) / eb, eb, 0, st>>>(d, chunks, P, A, b, sum_weight);
    k_cb_solve<<<1, kSolveThreads, cb_solve_smem(d), st>>>(d, (float)c.l2_reg_lambda, (float)c.gamma, c.discount_interval, A, b,
                                                           sum_weight, last_discount, inv_A, coefs, round_idx);
    launches_per_round = L.count + extra + 3;
    return PRL_OK;
}

extern "C" int prl_nlb_learn(prl_nlb *s, prl_buf *buf, int rounds, int batch, float *out_pred, float *out_label, float *out_weight,
                             float *out_loss, float *out_mu, int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && out_pred && out_loss && out_mu, "null argument");
    PRL_REQUIRE(s->cfg.action_rep != 0 || s->cfg.action_dim == 0,
                "learn over a buffer needs the state alone (action_dim 0) or a one-hot or binary action representation");
    NlCall call{};
    call.out_pred = out_pred; call.out_label = out_label; call.out_weight = out_weight; call.out_loss = out_loss; call.out_mu = out_mu;
    s->zero_weight = 0;
    return prl_nlb::learn(s, buf, rounds, batch, 0, out_logical, call, stream_);
}

extern "C" int prl_nlb_learn_batch(prl_nlb *s, int batch, const float *state, const float *action, const float *reward,
                                   const float *weight, int zero_weight, float *out_pred, float *out_loss, float *out_mu, void *stream_) {
    PRL_REQUIRE(s && (state || s->cfg.obs_dim == 0) && (action || s->cfg.action_dim == 0) && reward && out_pred && out_loss && out_mu,
                "null argument");
    NlCall dense{};
    dense.d_state = state; dense.d_action = action; dense.d_reward = reward; dense.d_weight = weight;
    dense.d_action_ld = s->cfg.action_dim;
    dense.out_pred = out_pred; dense.out_loss = out_loss; dense.out_mu = out_mu;
    s->zero_weight = zero_weight ? 1 : 0;
    const int rc = prl_nlb::learn_batch(s, batch, 0, dense, stream_);
    if (rc == PRL_OK && s->zero_weight) s->adam_step -= 1;   // no optimizer step
    s->zero_weight = 0;
    return rc;
}

extern "C" int prl_nlb_scores(prl_nlb *s, int n, const float *state, int n_space, const float *act_feat, double alpha, int mode,
                              const uint8_t *mask, float *out_scores, int32_t *out_index, void *stream_) {
    PRL_REQUIRE(s && out_scores && (state || s->cfg.obs_dim == 0) && (act_feat || s->cfg.action_dim == 0), "null argument");
    PRL_REQUIRE(n >= 0 && n_space >= 1 && (int64_t)n * n_space < ((int64_t)1 << 31), "n * n_space must be in [0, 2^31)");
    PRL_REQUIRE(mode >= 0 && mode <= 2, "mode must be 0 (act), 1 (get_scores) or 2 (get_scores, separate uncertainty)");
    if (n == 0) return PRL_OK;
    const prl_nlb_cfg &c = s->cfg;
    cudaStream_t st = (cudaStream_t)stream_;
    const long long total = (long long)n * n_space;
    const NlHead h = s->head();
    GemmLauncher L; L.st = st;
    for (long long r0 = 0; r0 < total; r0 += s->rows) {
        const int m = (int)(total - r0 < s->rows ? total - r0 : s->rows);
        k_cb_feat<<<(m * 32 + 255) / 256, 256, 0, st>>>(m, r0, n_space, c.obs_dim, c.action_dim, state, act_feat, s->X);
        s->forward(L, m);
        k_nl_scores<<<(m + 7) / 8, 256, 0, st>>>(m, r0, h, s->N, s->w + s->net.P, s->inv_A, s->coefs, mode, (float)alpha, out_scores);
    }
    if (out_index) k_cb_argmax<<<(n + 255) / 256, 256, 0, st>>>(n, n_space, out_scores, mask, out_index);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}

extern "C" int prl_nlb_ts_scores(prl_nlb *s, int n, const float *state, int n_space, const float *act_feat, const float *theta,
                                 int activate, const uint8_t *mask, float *out_scores, int32_t *out_index, void *stream_) {
    PRL_REQUIRE(s && theta && out_scores && (state || s->cfg.obs_dim == 0) && (act_feat || s->cfg.action_dim == 0), "null argument");
    PRL_REQUIRE(n >= 0 && n_space >= 1 && (int64_t)n * n_space < ((int64_t)1 << 31), "n * n_space must be in [0, 2^31)");
    if (n == 0) return PRL_OK;
    const prl_nlb_cfg &c = s->cfg;
    cudaStream_t st = (cudaStream_t)stream_;
    const long long total = (long long)n * n_space;
    const NlHead h = s->head();
    GemmLauncher L; L.st = st;
    for (long long r0 = 0; r0 < total; r0 += s->rows) {
        const int m = (int)(total - r0 < s->rows ? total - r0 : s->rows);
        k_cb_feat<<<(m * 32 + 255) / 256, 256, 0, st>>>(m, r0, n_space, c.obs_dim, c.action_dim, state, act_feat, s->X);
        s->forward(L, m);
        k_nl_ts_scores<<<(m * 32 + 255) / 256, 256, 0, st>>>(m, r0, h, s->N, theta, activate, out_scores);
    }
    if (out_index) k_cb_argmax<<<(n + 255) / 256, 256, 0, st>>>(n, n_space, out_scores, mask, out_index);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}
