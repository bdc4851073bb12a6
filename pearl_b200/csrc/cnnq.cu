// cnnq.cu — DQN / DoubleDQN on image observations (DeepQLearning / DoubleDQN built with CNNQValueNetwork or
// CNNQValueMultiHeadNetwork), driven by PolicyLearner.learn or called directly on a caller's batch (PearlAgent.learn_batch
// / offline_learning), replacing
//   neural_networks/sequential_decision_making/q_value_networks.py   CNNQValueNetwork (conv trunk on state / 255, the
//       features in (c, h, w) order concatenated with the one-hot action, FC stack with one output) and
//       CNNQValueMultiHeadNetwork (the FC stack on the features alone, one output per action; get_q_values = bmm with
//       the one-hot slots)
//   neural_networks/common/utils.py                                   conv_block (Conv2d + ReLU per layer, the last one
//       included), mlp_block
//   policy_learners/sequential_decision_making/deep_td_learning.py   forward, loss, learn_batch (target update FIRST,
//       MSE Bellman loss, AdamW step, reported mean |q - y|)
//   policy_learners/sequential_decision_making/deep_q_learning.py    get_next_state_values (max over available slots)
//   policy_learners/sequential_decision_making/double_dqn.py         get_next_state_values (online first argmax, target value)
//
// Round: the soft target update in flagged rounds (with the CURRENT online parameters, before anything else); the target
// net on the B next states; the online net on the B states (for DoubleDQN stacked with the B next states into one 2B-image
// pass); the head; the backward pass over the B state rows; AdamW(amsgrad); the report.  The target runs first because
// both passes share the trunk's im2col and activation buffers and the online pass's must survive to the backward pass.
// Fixed launch sequence, captured once per (batch, buffer) into a CUDA graph and replayed (DESIGN.md §3).
//
// Trunk: each conv layer is an explicit im2col of its input (rows (b, oh, ow), features (c, kh, kw): torch's
// [OC][C*KH*KW] weight layout) and one GemmLauncher product with bias and ReLU; layer 1's im2col divides the pixel values
// by 255 as the reference does (a true fp32 division).  Activations are kept as [(b, h, w)][c]; the last layer's are
// transposed into the reference's (c, h, w) feature order.  Backward-data is dY W followed by a gather col2im (every input
// element sums its (kh, kw) contributions in ascending order, masked by the ReLU of the layer below; no atomics).  The
// weight gradient contracts over B*OH*OW rows into a small [OC][C*K*K + 1] block, so its rows are split into S equal
// slices (S from the shape, split_of) launched as S stacked networks of one product, and the partial blocks are added in
// slice order.  Rows past B*OH*OW up to S slices are zero in dY (and in the im2col, except in DoubleDQN's stacked pass,
// where they hold next-state columns, finite values multiplied by those zeros).  The conv products use the tensor-core
// tiles (engine 2) unless the library's engine is the SIMT one.
//
// Head of row b:  V = max over available next slots k of Q'(s'_b)[id_k] (DQN), or Q'(s'_b)[id_k*] with k* the first
// argmax of Q(s'_b)[id_k] (DoubleDQN);  y_b = V gamma (1 - terminated) + r;  q_b = Q(s_b)[a_b].
//   CNNQValueNetwork: the one-hot fold, layer 1 = W1f feat + W1[:, F + a] + b1 (the feature product once per state, the
//     column add per action); dq_b = fl(2 / B)(q_b - y_b), reported mean_b |q_b - y_b|.
//   CNNQValueMultiHeadNetwork: the reference's get_q_values returns [B, 1] for the taken actions (it rebinds action_batch
//     to its 3-D form before its last shape test), and so does DoubleDQN's target lookup of one action per row, so its
//     MSELoss broadcasts to [B, B] pairs with targets Y_ij = y_j (DQN) or V_i gamma (1 - terminated_j) + r_j (DoubleDQN).
//     Reproduced: dq_i = sum_j fl(2 / B^2)(q_i - Y_ij), j ascending, on head column a_i; reported mean_{i,j} |q_i - Y_ij|.
// fp32, fixed summation order, no float atomics: bit-reproducible run to run and between graph replay and eager launches.
#include <limits.h>
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "rounds.cuh"
#include "gemm.cuh"
#include "qrows.cuh"

extern "C" int prl_get_contraction_engine(void);

using namespace prl;

namespace {

constexpr int kMaxA = 255;   // next-action ids are stored as bytes
constexpr int kMaxConv = 4, kMaxFc = 2, kMaxSplit = 64;

struct CnnqCall : QSetCall {};

// one block row per transition b (blockIdx.y): the blocks copy the state and next-state pixels; warp 0 of block column 0
// loads the rest of the row (reward, terminated, action, next-action ids) through load_row
__global__ void __launch_bounds__(256) k_cnnq_load(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int A, int dynamic,
                                                   const CnnqCall *__restrict__ call, const int *__restrict__ round_idx, int B,
                                                   float *__restrict__ S, float *__restrict__ S2, float *__restrict__ R,
                                                   float *__restrict__ T, int *__restrict__ act, int *__restrict__ cnt,
                                                   int *__restrict__ ids) {
    const int b = blockIdx.y;
    const uint32_t *rec = records ? records + (size_t)call->slots[(size_t)(*round_idx) * B + b] * L.record_words : nullptr;
    float *s = S + (size_t)b * obs, *s2 = S2 + (size_t)b * obs;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < obs; p += gridDim.x * blockDim.x) {
        if (rec) {
            s[p] = __uint_as_float(rec[L.off_state + p]);
            s2[p] = __uint_as_float(rec[L.off_next_state + p]);
        } else {
            s[p] = call->d_state[(size_t)b * obs + p];
            s2[p] = call->d_next_state[(size_t)b * obs + p];
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < 32) {
        const QRow row = load_row<true>(records, L, 0, A, dynamic, call, round_idx, B, b, threadIdx.x, S, S2, R, T, ids);
        if (threadIdx.x == 0) {
            act[b] = row.action;
            cnt[b] = row.cnt;
        }
    }
}

// col[r][f], r = (b, oh, ow) < rows, f = (c, kh, kw) < C K K: the layer input under the window, zero in the padding.
// nchw: the input is the state batch [b][c][h][w] of pixel values, divided by 255 (layer 1); otherwise the previous
// layer's activations [(b, h, w)][c].  Rows in [rows, total / (C K K)) are zero.
__global__ void k_im2col(int64_t total, int rows, int C, int H, int W, int K, int stride, int pad, int OH, int OW, int nchw,
                         const float *__restrict__ x, float *__restrict__ col) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int KK = C * K * K;
    const int r = (int)(e / KK), f = (int)(e - (int64_t)r * KK);
    float v = 0.f;
    if (r < rows) {
        const int b = r / (OH * OW), p = r - b * OH * OW, oh = p / OW, ow = p - oh * OW;
        const int c = f / (K * K), q = f - c * K * K, kh = q / K, kw = q - kh * K;
        const int ih = oh * stride - pad + kh, iw = ow * stride - pad + kw;
        if (ih >= 0 && ih < H && iw >= 0 && iw < W)
            v = nchw ? __fdiv_rn(x[(((size_t)b * C + c) * H + ih) * W + iw], 255.f) : x[(((size_t)b * H + ih) * W + iw) * C + c];
    }
    col[e] = v;
}

// dx[r][c], r = (b, ih, iw) < rows: the sum over (kh, kw), kh then kw ascending, of dcol[(b, oh, ow)][(c, kh, kw)] for
// every output position whose window covers (ih, iw), kept only where act[r][c] > 0 (the ReLU of the layer below).
// Rows in [rows, total / C) are zero.
__global__ void k_col2im(int64_t total, int rows, int C, int H, int W, int K, int stride, int pad, int OH, int OW,
                         const float *__restrict__ dcol, const float *__restrict__ act, float *__restrict__ dx) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int r = (int)(e / C), c = (int)(e - (int64_t)r * C);
    float s = 0.f;
    if (r < rows && act[e] > 0.f) {
        const int b = r / (H * W), p = r - b * H * W, ih = p / W, iw = p - ih * W;
        const int KK = C * K * K;
        for (int kh = 0; kh < K; kh++) {
            const int th = ih + pad - kh;
            if (th < 0 || th % stride) continue;
            const int oh = th / stride;
            if (oh >= OH) continue;
            for (int kw = 0; kw < K; kw++) {
                const int tw = iw + pad - kw;
                if (tw < 0 || tw % stride) continue;
                const int ow = tw / stride;
                if (ow >= OW) continue;
                s += dcol[(((size_t)b * OH + oh) * OW + ow) * KK + (c * K + kh) * K + kw];
            }
        }
    }
    dx[e] = s;
}

// feat[b][c HW + p] = y[b HW + p][c]: the last layer's activations in the reference's view(B, -1) order
__global__ void k_to_feat(int64_t total, int HW, int C, const float *__restrict__ y, float *__restrict__ feat) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int64_t b = e / ((int64_t)C * HW);
    const int rem = (int)(e - b * C * HW), c = rem / HW, p = rem - c * HW;
    feat[e] = y[((size_t)b * HW + p) * C + c];
}

// dy[r][c] = dfeat[b][c HW + p] for r = b HW + p < rows; zero for the rows up to total / C
__global__ void k_from_feat(int64_t total, int rows, int HW, int C, const float *__restrict__ dfeat, float *__restrict__ dy) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int r = (int)(e / C), c = (int)(e - (int64_t)r * C);
    float v = 0.f;
    if (r < rows) {
        const int b = r / HW, p = r - b * HW;
        v = dfeat[((size_t)b * C + c) * HW + p];
    }
    dy[e] = v;
}

// dst[j] = sum over slices z = 0, 1, ... of the split contraction's partial gradients: the weights part[z][j] (j < nw),
// then the biases part[S nw + z nb + j - nw]
__global__ void k_slice_sum(int nw, int nb, int S, const float *__restrict__ part, float *__restrict__ dst) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= nw + nb) return;
    const float *p = j < nw ? part + j : part + (size_t)S * nw + (j - nw);
    const int step = j < nw ? nw : nb;
    float s = 0.f;
    for (int z = 0; z < S; z++) s += p[(size_t)z * step];
    dst[j] = s;
}

// the one-hot fold of CNNQValueNetwork's first FC layer: out[row][j] = act(P[b][j] + W0[j][F + id]) for row = b n + k,
// id = ids[row] (n = 1: the taken actions) or k (ids null: slot k holds action k); act = ReLU unless it is the last layer
__global__ void k_cnn_fold(int64_t total, int n, int Z, const float *__restrict__ P, const float *__restrict__ w0a, int ld,
                           const int *__restrict__ ids, int relu, float *__restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int row = (int)(e / Z), j = (int)(e - (int64_t)row * Z), b = row / n, k = row - b * n;
    const int id = ids ? ids[row] : k;
    const float v = P[(size_t)b * Z + j] + __ldg(w0a + (size_t)j * ld + id);
    out[e] = relu ? fmaxf(v, 0.f) : v;
}

// Bellman target and error of row b, one warp per row (lane l takes next slots l, l + 32, ...).  qa: the online values at
// the states, [B] at the taken actions (vanilla) or [B][A] (multi-head); qn / qt: [B][A] online / target values at s'.
// Vanilla: dq[b] = fl(2 / B)(q_b - y_b), rowabs[b] = |q_b - y_b|.  Multi-head: q_b, y_b and V_b into qv / yv / vv
// (k_cnnq_bcast).
__global__ void __launch_bounds__(128) k_cnnq_head(int B, int A, int dbl, int multi, const float *__restrict__ qa,
                                                   const float *__restrict__ qn, const float *__restrict__ qt,
                                                   const int *__restrict__ ids, const int *__restrict__ cnt,
                                                   const int *__restrict__ act, const float *__restrict__ term,
                                                   const float *__restrict__ rew, float gamma, float *__restrict__ qv,
                                                   float *__restrict__ yv, float *__restrict__ vv, float *__restrict__ dq,
                                                   float *__restrict__ rowabs) {
    const int lane = threadIdx.x & 31, b = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (b >= B) return;
    const int n_ok = cnt[b];
    const int *nid = ids + (size_t)b * A;
    const float *sel = (dbl ? qn : qt) + (size_t)b * A;
    float best = -INFINITY;
    int bk = INT_MAX;
    for (int k = lane; k < A; k += 32) {
        const float v = k < n_ok ? sel[nid[k]] : -INFINITY;
        if (v > best || (v == best && k < bk)) { best = v; bk = k; }
    }
    warp_first_max(best, bk);
    if (lane) return;
    const float V = dbl ? qt[(size_t)b * A + nid[bk == INT_MAX ? 0 : bk]] : best;
    const float y = __fadd_rn(__fmul_rn(__fmul_rn(V, gamma), __fsub_rn(1.f, term[b])), rew[b]);
    const float q = multi ? qa[(size_t)b * A + act[b]] : qa[b];
    if (multi) {
        qv[b] = q;
        yv[b] = y;
        vv[b] = V;
    } else {
        const float e = __fsub_rn(q, y);
        dq[b] = __fmul_rn(__fdiv_rn(2.f, (float)B), e);
        rowabs[b] = fabsf(e);
    }
}

// multi-head: the B x B broadcast of the reference's MSELoss (file header), one thread per row i, over the pair targets
//   Y_ij = y_j (DQN),  V_i gamma (1 - terminated_j) + r_j (DoubleDQN):
//   dQ[i][j] = [j = a_i] sum_j' fl(2 / B^2)(q_i - Y_ij'),  rowabs[i] = (sum_j' |q_i - Y_ij'|) / B,  j' ascending
__global__ void k_cnnq_bcast(int B, int A, int dbl, float gamma, const float *__restrict__ qv, const float *__restrict__ yv,
                             const float *__restrict__ vv, const float *__restrict__ term, const float *__restrict__ rew,
                             const int *__restrict__ act, float *__restrict__ dq, float *__restrict__ rowabs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B) return;
    const float q = qv[i], c = __fdiv_rn(2.f, __fmul_rn((float)B, (float)B)), vg = __fmul_rn(vv[i], gamma);
    float g = 0.f, a = 0.f;
    for (int j = 0; j < B; j++) {
        const float Y = dbl ? __fadd_rn(__fmul_rn(vg, __fsub_rn(1.f, term[j])), rew[j]) : yv[j];
        const float e = __fsub_rn(q, Y);
        g = __fadd_rn(g, __fmul_rn(c, e));
        a = __fadd_rn(a, fabsf(e));
    }
    const int ai = act[i];
    float *d = dq + (size_t)i * A;
    for (int j = 0; j < A; j++) d[j] = j == ai ? g : 0.f;
    rowabs[i] = __fdiv_rn(a, (float)B);
}

inline unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace

// ------------------------------------------------------------------ host side
struct prl_cnnq : FlatQ<prl_cnnq, CnnqCall, prl_cnnq_cfg> {
    static constexpr const char *kFn = "prl_cnnq", *kName = "CNN DQN";
    static constexpr int kGraphs = 3;
    // shapes: conv layer l maps [ci][hi][wi] to [co][ho][wo] with a k x k kernel (kk = ci k k features); FC layer i maps
    // fd[i] to fd[i + 1] (fd[0] = F features, fd[nf + 1] = 1 or A outputs); layer 0's weight row has ld0 = F (+ A) entries
    int nc, nf, obs, F, ld0;
    int ci[kMaxConv], hi[kMaxConv], wi[kMaxConv], co[kMaxConv], ho[kMaxConv], wo[kMaxConv], k[kMaxConv], sd[kMaxConv], pd[kMaxConv],
        kk[kMaxConv];
    int fd[kMaxFc + 2];
    int Wc[kMaxConv], bc[kMaxConv], Wf[kMaxFc + 1], bf[kMaxFc + 1];
    // workspace: S holds the states and, right after the round's B rows, the next states (one 2B-image online pass)
    float *S, *R, *T, *col[kMaxConv], *y[kMaxConv], *dy[kMaxConv], *dcol, *part, *feat, *dfeat, *pf, *fo[kMaxFc], *fx[kMaxFc],
        *dfc[kMaxFc], *qo, *qn, *qt, *qv, *yv, *vv, *dq, *rowabs, *grad;
    int *act, *cnt, *ids;
    static int check(const prl_cnnq_cfg *c);
    static int64_t layout(prl_cnnq *s);
    static int64_t carve(prl_cnnq *s, void *base);
    static int round(prl_cnnq *s, prl_buf *buf, int B, cudaStream_t st);
    int buffer_ok(const prl_buf *buf) const {
        PRL_REQUIRE((buf->desc.flags & PRL_BUF_DISCRETE) && buf->desc.obs_dim == obs && buf->desc.n_actions == cfg.n_actions,
                    "%s needs a discrete-action buffer with obs_dim = in_c * in_h * in_w = %d and n_actions = %d", kName, obs, cfg.n_actions);
        PRL_REQUIRE(buf->shard_world <= 1, "the buffer is one shard of a multi-GPU buffer: %s samples local buffers only", kName);
        return PRL_OK;
    }
};

namespace {

// slices of a conv layer's weight-gradient contraction over R rows into [OC][KK + 1]: about two CTAs per SM of the
// 128 x 64 tensor-core tiles, slices of at least 128 rows, at most kMaxSplit
int split_of(int64_t R, int OC, int KK) {
    const int64_t tiles = (int64_t)((OC + 127) / 128) * ((KK + 1 + 63) / 64);
    int64_t S = 264 / tiles;
    if (S > R / 128) S = R / 128;
    if (S > kMaxSplit) S = kMaxSplit;
    return S < 1 ? 1 : (int)S;
}

// the rows the weight-gradient contraction of layer l reads at batch B (S slices of equal length, zero-padded)
int64_t padded_rows(const prl_cnnq *s, int l, int B, int *S_out = nullptr, int *slice_out = nullptr) {
    const int64_t R = (int64_t)B * s->ho[l] * s->wo[l];
    const int S = split_of(R, s->co[l], s->kk[l]);
    const int64_t slice = (R + S - 1) / S;
    if (S_out) *S_out = S;
    if (slice_out) *slice_out = (int)slice;
    return slice * S;
}

}  // namespace

// the shapes, the parameter offsets and P, set when the count stays below 2^31; returns the count (-1: a conv output
// would be empty)
int64_t prl_cnnq::layout(prl_cnnq *s) {
    const prl_cnnq_cfg &c = s->cfg;
    s->nc = c.n_conv; s->nf = c.n_fc;
    s->obs = c.in_c * c.in_h * c.in_w;
    int C = c.in_c, H = c.in_h, W = c.in_w;
    int64_t o = 0;
    for (int l = 0; l < s->nc; l++) {
        s->ci[l] = C; s->hi[l] = H; s->wi[l] = W;
        s->co[l] = c.conv_out[l]; s->k[l] = c.conv_kernel[l]; s->sd[l] = c.conv_stride[l]; s->pd[l] = c.conv_pad[l];
        const int eh = H + 2 * s->pd[l] - s->k[l], ew = W + 2 * s->pd[l] - s->k[l];
        if (eh < 0 || ew < 0) return -1;
        s->ho[l] = eh / s->sd[l] + 1; s->wo[l] = ew / s->sd[l] + 1;
        s->kk[l] = C * s->k[l] * s->k[l];
        s->Wc[l] = (int)o; o += (int64_t)s->co[l] * s->kk[l];
        s->bc[l] = (int)o; o += s->co[l];
        C = s->co[l]; H = s->ho[l]; W = s->wo[l];
        if (o >= ((int64_t)1 << 31)) return o;
    }
    s->F = C * H * W;
    s->fd[0] = s->F;
    for (int i = 0; i < s->nf; i++) s->fd[i + 1] = c.fc_hidden[i];
    s->fd[s->nf + 1] = c.multi_head ? c.n_actions : 1;
    s->ld0 = s->F + (c.multi_head ? 0 : c.n_actions);
    for (int i = 0; i <= s->nf; i++) {
        const int in = i == 0 ? s->ld0 : s->fd[i];
        s->Wf[i] = (int)o; o += (int64_t)s->fd[i + 1] * in;
        s->bf[i] = (int)o; o += s->fd[i + 1];
        if (o >= ((int64_t)1 << 31)) return o;
    }
    s->P = (int)o;
    return o;
}

int prl_cnnq::check(const prl_cnnq_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->in_c > 0 && c->in_h > 0 && c->in_w > 0, "the input channels, height and width must be positive");
    PRL_REQUIRE(c->n_conv >= 1 && c->n_conv <= kMaxConv, "n_conv must be in [1, %d]", kMaxConv);
    for (int l = 0; l < c->n_conv; l++)
        PRL_REQUIRE(c->conv_out[l] > 0 && c->conv_kernel[l] > 0 && c->conv_stride[l] > 0 && c->conv_pad[l] >= 0,
                    "conv layer %d: out-channels, kernel and stride must be positive and the padding non-negative", l);
    PRL_REQUIRE(c->n_fc >= 0 && c->n_fc <= kMaxFc, "n_fc (hidden fully connected layers) must be in [0, %d]", kMaxFc);
    for (int i = 0; i < c->n_fc; i++) PRL_REQUIRE(c->fc_hidden[i] > 0, "fc_hidden[%d] must be positive", i);
    PRL_REQUIRE(c->n_actions >= 1 && c->n_actions <= kMaxA, "n_actions must be in [1, %d]: next-action ids are stored as bytes", kMaxA);
    PRL_REQUIRE(c->target_update_freq > 0, "target_update_freq must be positive");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    prl_cnnq t; t.cfg = *c;
    const int64_t P = layout(&t);
    PRL_REQUIRE(P >= 0, "a conv layer's output would be empty: every conv output must be at least 1 x 1");
    PRL_REQUIRE(P < ((int64_t)1 << 31), "the parameter count %lld must stay below 2^31 (32-bit element offsets)", (long long)P);
    // the largest buffers a product or kernel indexes with 32-bit element offsets: the im2col and activations of the
    // stacked 2 max_batch-image pass (plus the split's padding rows), the states, and the FC rows of every action slot
    const int64_t B = c->max_batch, M = 2 * B, A = c->n_actions;
    int64_t big = M * t.obs;
    for (int l = 0; l < t.nc; l++) {
        const int64_t rows = M * t.ho[l] * t.wo[l] + kMaxSplit;
        big = std::max(big, std::max(rows * t.kk[l], rows * (int64_t)t.co[l]));
    }
    for (int i = 0; i <= t.nf + 1; i++) big = std::max(big, std::max(M, B * A) * (int64_t)std::max(t.fd[i], t.ld0));
    PRL_REQUIRE(big < ((int64_t)1 << 31),
                "the largest im2col / activation buffer (%lld elements at max_batch = %d) must stay below 2^31 (32-bit element offsets)",
                (long long)big, c->max_batch);
    return PRL_OK;
}

// the workspace, in order; base == null: only its size
int64_t prl_cnnq::carve(prl_cnnq *s, void *base) {
    const prl_cnnq_cfg &c = s->cfg;
    const int64_t B = c.max_batch, M = c.double_dqn ? 2 * B : B, A = c.n_actions, BA = B * A, Z0 = s->fd[1];
    Carve w{(char *)base};
    w(s->S, 2 * B * s->obs); w(s->R, B); w(s->T, B);
    int64_t dcol = 0, part = 0;
    for (int l = 0; l < s->nc; l++) {
        const int64_t rows = M * s->ho[l] * s->wo[l] + kMaxSplit;   // the split pads fewer than kMaxSplit rows
        w(s->col[l], rows * s->kk[l]); w(s->y[l], rows * s->co[l]); w(s->dy[l], rows * s->co[l]);
        dcol = std::max(dcol, B * s->ho[l] * s->wo[l] * (int64_t)s->kk[l]);
        int S = 1;
        padded_rows(s, l, (int)B, &S);
        part = std::max(part, (int64_t)S * s->co[l] * (s->kk[l] + 1));
    }
    w(s->dcol, dcol); w(s->part, part);
    w(s->feat, M * s->F); w(s->dfeat, B * s->F); w(s->pf, M * Z0);
    for (int i = 0; i < s->nf; i++) {
        w(s->fo[i], M * s->fd[i + 1]); w(s->fx[i], std::max(BA, M) * s->fd[i + 1]); w(s->dfc[i], B * s->fd[i + 1]);
    }
    w(s->qo, M * A); w(s->qn, BA); w(s->qt, BA); w(s->qv, B); w(s->yv, B); w(s->vv, B); w(s->dq, BA); w(s->rowabs, B); w(s->grad, s->P);
    w(s->act, B); w(s->cnt, B); w(s->ids, BA);
    s->carve_tail(w, c.max_rounds, B);
    return w.bytes;
}

extern "C" int64_t prl_cnnq_param_count(const prl_cnnq_cfg *c) { return prl_cnnq::param_count(c); }
extern "C" int64_t prl_cnnq_workspace_bytes(const prl_cnnq_cfg *c) { return prl_cnnq::workspace_bytes(c); }
extern "C" int prl_cnnq_create(prl_cnnq **out, const prl_cnnq_cfg *cfg, float *w, float *w_target, float *exp_avg, float *exp_avg_sq,
                               float *max_exp_avg_sq, int64_t adam_step, void *workspace) {
    return prl_cnnq::create(out, cfg, w, w_target, exp_avg, exp_avg_sq, max_exp_avg_sq, adam_step, workspace);
}
extern "C" int prl_cnnq_destroy(prl_cnnq *s) { return prl_cnnq::destroy(s); }
extern "C" int64_t prl_cnnq_adam_step(const prl_cnnq *s) { return prl_cnnq::adam_step_of(s); }
extern "C" int prl_cnnq_set_adam_step(prl_cnnq *s, int64_t step) { return prl_cnnq::set_adam_step(s, step); }
extern "C" int prl_cnnq_set_lr(prl_cnnq *s, double lr) { return prl_cnnq::set_lr(s, lr); }
extern "C" int prl_cnnq_set_graph(prl_cnnq *s, int enable) { return prl_cnnq::set_graph(s, enable); }
extern "C" int64_t prl_cnnq_last_launches(const prl_cnnq *s) { return prl_cnnq::last_launches_of(s); }

namespace {

constexpr int kEb = 256;

// the products of the trunk: the tensor-core tiles, unless the library runs the SIMT ones
int conv_engine() { return prl_get_contraction_engine() == 0 ? 0 : 2; }

// the conv trunk of `net` on m images x ([m][C][H][W] pixel values) into feat [m][F]; B > 0: the round's batch, whose
// weight-gradient rows past B OH OW are zeroed in the im2col when the pass does not cover them
void trunk(const prl_cnnq *s, GemmLauncher &L, const float *net, const float *x, int m, int B, int &small) {
    const int saved = L.engine;
    L.engine = conv_engine();
    for (int l = 0; l < s->nc; l++) {
        const int64_t rows = (int64_t)m * s->ho[l] * s->wo[l];
        const int64_t padded = std::max(rows, B > 0 ? padded_rows(s, l, B) : rows);
        const int64_t total = padded * s->kk[l];
        k_im2col<<<blocks(total, kEb), kEb, 0, L.st>>>(total, (int)rows, s->ci[l], s->hi[l], s->wi[l], s->k[l], s->sd[l], s->pd[l], s->ho[l],
                                                       s->wo[l], l == 0, l == 0 ? x : s->y[l - 1], s->col[l]);
        L.fwd(mat(s->col[l], s->kk[l]), (int)rows, net + s->Wc[l], s->kk[l], 0, net + s->bc[l], 0, s->co[l], s->kk[l], true, s->y[l],
              s->co[l], 0);
        small++;
    }
    L.engine = saved;
    const int last = s->nc - 1, HW = s->ho[last] * s->wo[last];
    const int64_t total = (int64_t)m * s->F;
    k_to_feat<<<blocks(total, kEb), kEb, 0, L.st>>>(total, HW, s->co[last], s->y[last], s->feat);
    small++;
}

// FC layers 1..nf of `net` on m rows whose layer-0 output is h[0]: a_2 .. a_nf into h[1..nf), the outputs into out
void fc_rest(const prl_cnnq *s, GemmLauncher &L, const float *net, int m, float *const *h, float *out) {
    for (int i = 1; i <= s->nf; i++)
        L.fwd(mat(h[i - 1], s->fd[i]), m, net + s->Wf[i], s->fd[i], 0, net + s->bf[i], 0, s->fd[i + 1], s->fd[i], i < s->nf,
              i < s->nf ? h[i] : out, s->fd[i + 1], 0);
}

// multi-head: the FC stack of `net` on m feature rows (feat), hidden activations into h, the A head values into out
void fc_multi(const prl_cnnq *s, GemmLauncher &L, const float *net, const float *feat, int m, float *const *h, float *out) {
    L.fwd(mat(feat, s->F), m, net + s->Wf[0], s->ld0, 0, net + s->bf[0], 0, s->fd[1], s->F, s->nf > 0, s->nf > 0 ? h[0] : out,
          s->fd[1], 0);
    fc_rest(s, L, net, m, h, out);
}

// vanilla: layer 0's feature product pf = feat W0[:, :F]^T + b0 on m rows (no activation: the action column comes next)
void fc_p(const prl_cnnq *s, GemmLauncher &L, const float *net, const float *feat, int m) {
    L.fwd(mat(feat, s->F), m, net + s->Wf[0], s->ld0, 0, net + s->bf[0], 0, s->fd[1], s->F, false, s->pf, s->fd[1], 0);
}

// vanilla: the fold of n slots per row of pf (from row p0 on; ids as k_cnn_fold), then the rest of the stack; the m n
// values into out
void fc_fold(const prl_cnnq *s, GemmLauncher &L, const float *net, int p0, int m, int n, const int *ids, float *const *h, float *out,
             int &small) {
    const int Z = s->fd[1];
    const int64_t total = (int64_t)m * n * Z;
    k_cnn_fold<<<blocks(total, kEb), kEb, 0, L.st>>>(total, n, Z, s->pf + (size_t)p0 * Z, net + s->Wf[0] + s->F, s->ld0, ids, s->nf > 0,
                                                     s->nf > 0 ? h[0] : out);
    small++;
    fc_rest(s, L, net, m * n, h, out);
}

// Q(s)[a] for every action of `net` on m rows of feat into out [m][A]
void q_all(const prl_cnnq *s, GemmLauncher &L, const float *net, int p0, const float *feat, int m, float *out, int &small) {
    float *const *scratch = s->fx;
    if (s->cfg.multi_head) fc_multi(s, L, net, feat, m, scratch, out);
    else fc_fold(s, L, net, p0, m, s->cfg.n_actions, nullptr, scratch, out, small);
}

}  // namespace

// one learner round, launched (or captured) on `st`; buf == null: the dense batch of the call block (learn_batch)
int prl_cnnq::round(prl_cnnq *s, prl_buf *buf, int B, cudaStream_t st) {
    const prl_cnnq_cfg &c = s->cfg;
    const int A = c.n_actions, multi = c.multi_head, dbl = c.double_dqn, F = s->F, Z0 = s->fd[1];
    // the decay factor is overridden by call->decay (k_adamw's decay pointer)
    const AdamHp h = adam_hp(0.0, c.beta1, c.beta2, c.eps, c.weight_decay);
    GemmLauncher L; L.st = st;
    const float *w = s->q;
    float *g = s->grad, *S2 = s->S + (size_t)B * s->obs;
    int small = 0;
    const int dynamic = (buf && (buf->desc.flags & PRL_BUF_DYNAMIC_ACTIONS)) ? 1 : 0;
    k_cnnq_load<<<dim3(std::min((s->obs + 1023) / 1024, 64), B), kEb, 0, st>>>(buf ? buf->records : nullptr, buf ? buf->lay : prl_buf_layout{},
                                                                            s->obs, A, dynamic, s->call, s->round_idx, B, s->S, S2, s->R,
                                                                            s->T, s->act, s->cnt, s->ids);
    // ---------------- target update first, with the current online parameters (flagged rounds only)
    k_soft_update_flagged<<<blocks(s->P, kEb), kEb, 0, st>>>(s->P, s->q, s->q_t, (float)c.tau, (float)(1.0 - c.tau), s->target_on,
                                                            s->round_idx);
    small += 2;
    // ---------------- the target net on the next states
    trunk(s, L, s->q_t, S2, B, 0, small);
    if (!multi) fc_p(s, L, s->q_t, s->feat, B);
    q_all(s, L, s->q_t, 0, s->feat, B, s->qt, small);
    // ---------------- the online net on the states (kept for the backward pass) and, for DoubleDQN, the next states: images
    // B..2B-1 of the same pass
    const int m = dbl ? 2 * B : B;
    trunk(s, L, w, s->S, m, B, small);
    const float *qn = s->qn;
    if (multi) {
        fc_multi(s, L, w, s->feat, m, s->fo, s->qo);
        qn = s->qo + (size_t)B * A;
    } else {
        fc_p(s, L, w, s->feat, m);
        fc_fold(s, L, w, 0, B, 1, s->act, s->fo, s->qo, small);
        if (dbl) q_all(s, L, w, B, s->feat + (size_t)B * F, B, s->qn, small);
    }
    // ---------------- Bellman target and the head gradient
    k_cnnq_head<<<(B + 3) / 4, 128, 0, st>>>(B, A, dbl, multi, s->qo, qn, s->qt, s->ids, s->cnt, s->act, s->T, s->R, (float)c.gamma,
                                             s->qv, s->yv, s->vv, s->dq, s->rowabs);
    small++;
    if (multi) {
        k_cnnq_bcast<<<blocks(B, 128), 128, 0, st>>>(B, A, dbl, (float)c.gamma, s->qv, s->yv, s->vv, s->T, s->R, s->act, s->dq, s->rowabs);
        small++;
    }
    // ---------------- backward through the FC stack over the B state rows
    const float *dcur = s->dq;
    for (int i = s->nf; i >= 1; i--) {
        const int no = s->fd[i + 1], ni = s->fd[i];
        L.bwd_w(dcur, no, 0, B, no, mat(s->fo[i - 1], ni), ni, g + s->Wf[i], ni, 0, g + s->bf[i], 0);
        L.bwd_x(dcur, no, 0, B, no, w + s->Wf[i], ni, 0, 0, ni, s->dfc[i - 1], ni, 0, s->fo[i - 1], ni, 0, false);
        dcur = s->dfc[i - 1];
    }
    L.bwd_w(dcur, Z0, 0, B, Z0, mat(s->feat, F), F, g + s->Wf[0], s->ld0, 0, g + s->bf[0], 0);
    if (!multi) {
        k_fold_w1a_grad<<<blocks((int64_t)Z0 * A, kEb), kEb, 0, st>>>(B, A, Z0, s->act, dcur, g + s->Wf[0] + F, s->ld0, 0);
        small++;
    }
    L.bwd_x(dcur, Z0, 0, B, Z0, w + s->Wf[0], s->ld0, 0, 0, F, s->dfeat, F, 0, s->feat, F, 0, false);
    // ---------------- backward through the trunk: the features back to [(b, h, w)][c], then per layer the split weight
    // gradient and, below layer 1, dY W and the gather col2im
    L.engine = conv_engine();
    {
        const int l = s->nc - 1;
        const int64_t total = padded_rows(s, l, B) * s->co[l];
        k_from_feat<<<blocks(total, kEb), kEb, 0, st>>>(total, B * s->ho[l] * s->wo[l], s->ho[l] * s->wo[l], s->co[l], s->dfeat, s->dy[l]);
        small++;
    }
    for (int l = s->nc - 1; l >= 0; l--) {
        const int OC = s->co[l], KK = s->kk[l], R = B * s->ho[l] * s->wo[l];
        int S = 1, slice = 0;
        padded_rows(s, l, B, &S, &slice);
        L.bwd_w(s->dy[l], OC, (long long)slice * OC, slice, OC, mat(s->col[l], KK, (long long)slice * KK), KK, s->part, KK,
                (long long)OC * KK, s->part + (size_t)S * OC * KK, OC, S);
        k_slice_sum<<<blocks((int64_t)OC * KK + OC, kEb), kEb, 0, st>>>(OC * KK, OC, S, s->part, g + s->Wc[l]);
        small++;
        if (l == 0) break;
        L.bwd_x(s->dy[l], OC, 0, R, OC, w + s->Wc[l], KK, 0, 0, KK, s->dcol, KK, 0, nullptr, 0, 0, false);
        const int64_t total = padded_rows(s, l - 1, B) * s->ci[l];
        k_col2im<<<blocks(total, kEb), kEb, 0, st>>>(total, B * s->hi[l] * s->wi[l], s->ci[l], s->hi[l], s->wi[l], s->k[l], s->sd[l], s->pd[l],
                                                     s->ho[l], s->wo[l], s->dcol, s->y[l - 1], s->dy[l - 1]);
        small++;
    }
    // ---------------- AdamW(amsgrad); the target was updated at the start of the round
    k_adamw<<<blocks(s->P, kEb), kEb, 0, st>>>(s->P, s->q, s->q_m, s->q_v, s->q_x, g, h, s->scal, s->round_idx, nullptr, 0.f, 0.f,
                                              &s->call->decay);
    k_round_report<<<1, 256, 0, st>>>(B, s->rowabs, s->call, s->round_idx);
    small += 2;
    s->launches_per_round = L.count + small;
    return PRL_OK;
}

extern "C" int prl_cnnq_learn(prl_cnnq *s, prl_buf *buf, int rounds, int batch, int64_t training_steps, float *out_loss,
                              int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(s && buf && out_loss, "null argument");
    CnnqCall call{};
    call.out_loss = out_loss;
    return prl_cnnq::learn(s, buf, rounds, batch, training_steps, out_logical, call, stream_);
}

extern "C" int prl_cnnq_learn_batch(prl_cnnq *s, int batch, const float *state, const int32_t *action_id, const float *reward,
                                    const float *next_state, const uint8_t *terminated, const int32_t *next_ids,
                                    const int32_t *next_count, int64_t training_steps, float *out_loss, void *stream_) {
    PRL_REQUIRE(s && state && action_id && reward && next_state && terminated && out_loss, "null argument");
    CnnqCall dense{};
    dense.d_state = state; dense.d_next_state = next_state; dense.d_reward = reward; dense.d_action_id = action_id;
    dense.d_next_ids = next_ids; dense.d_next_cnt = next_count; dense.d_term = terminated;
    dense.out_loss = out_loss;
    return prl_cnnq::learn_batch(s, batch, training_steps, dense, stream_);
}

// Q(s)[a] for every action: the online (or target) forward of the round on n images (chunks of max_batch images through
// the workspace)
extern "C" int prl_cnnq_q_values(prl_cnnq *s, int n, const float *state, int target, float *out_q, void *stream_) {
    PRL_REQUIRE(s && state && out_q, "null argument");
    if (n <= 0) return PRL_OK;
    const prl_cnnq_cfg &c = s->cfg;
    const float *w = target ? s->q_t : s->q;
    GemmLauncher L; L.st = (cudaStream_t)stream_;
    int small = 0;
    for (int r0 = 0; r0 < n; r0 += c.max_batch) {
        const int m = n - r0 < c.max_batch ? n - r0 : c.max_batch;
        trunk(s, L, w, state + (size_t)r0 * s->obs, m, 0, small);
        if (!c.multi_head) fc_p(s, L, w, s->feat, m);
        q_all(s, L, w, 0, s->feat, m, out_q + (size_t)r0 * c.n_actions, small);
    }
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}
