// ac_nets.cuh — the network pieces of the learners built on VanillaActorNetwork (softmax policy) and VanillaValueNetwork
// (ppo.cu, reinforce.cu): the flat parameter layout of a two-hidden-layer MLP, its forward pass and its backward chain as
// GemmLauncher contractions, and the read of the newest transition's next_state that the rollout's bootstrap value starts
// from.
#pragma once
#include "gemm.cuh"

namespace prl {

// Offsets into the flat fp32 vector of nn.Sequential(Linear, ReLU, Linear, ReLU, Linear) in torch's parameters() order:
// W1[h1][in] b1 W2[h2][h1] b2 W3[out][h2] b3 (row-major [out][in]); P = the parameter count
struct Mlp2 {
    int in, h1, h2, out;
    int W1, b1, W2, b2, W3, b3, P;
};
inline Mlp2 mlp2(int in, int h1, int h2, int out) {
    Mlp2 n{in, h1, h2, out};
    int o = 0;
    n.W1 = o; o += h1 * in; n.b1 = o; o += h1;
    n.W2 = o; o += h2 * h1; n.b2 = o; o += h2;
    n.W3 = o; o += out * h2; n.b3 = o; o += out;
    n.P = o;
    return n;
}

// X[rows][in] -> H1 = relu(X W1^T + b1), H2 = relu(H1 W2^T + b2), Y = H2 W3^T + b3: three contractions
inline void mlp2_forward(GemmLauncher &L, const Mlp2 &n, const float *w, const float *X, int rows, float *H1, float *H2, float *Y) {
    L.fwd(mat(X, n.in), rows, w + n.W1, n.in, 0, w + n.b1, 0, n.h1, n.in, true, H1, n.h1, 0);
    L.fwd(mat(H1, n.h1), rows, w + n.W2, n.h1, 0, w + n.b2, 0, n.h2, n.h1, true, H2, n.h2, 0);
    L.fwd(mat(H2, n.h2), rows, w + n.W3, n.h2, 0, w + n.b3, 0, n.out, n.h2, false, Y, n.out, 0);
}

// Parameter gradient g (every element written) of B rows from dY[B][out] and the forward activations X, H1, H2;
// dH2 / dH1 are scratch.  Four contractions, and dH2 as a fifth (out > 1) or as one k_head_bwd launch (a scalar head)
inline void mlp2_backward(GemmLauncher &L, const Mlp2 &n, const float *w, float *g, const float *dY, const float *X, const float *H1,
                          const float *H2, float *dH2, float *dH1, int B) {
    L.bwd_w(dY, n.out, 0, B, n.out, mat(H2, n.h2), n.h2, g + n.W3, n.h2, 0, g + n.b3, 0);
    if (n.out == 1) {
        const int eb = 256;
        k_head_bwd<<<dim3((B * n.h2 + eb - 1) / eb, 1, 1), eb, 0, L.st>>>(B, n.h2, dY, w + n.W3, 0, H2, dH2);
    } else {
        L.bwd_x(dY, n.out, 0, B, n.out, w + n.W3, n.h2, 0, 0, n.h2, dH2, n.h2, 0, H2, n.h2, 0, false);
    }
    L.bwd_w(dH2, n.h2, 0, B, n.h2, mat(H1, n.h1), n.h1, g + n.W2, n.h1, 0, g + n.b2, 0);
    L.bwd_x(dH2, n.h2, 0, B, n.h2, w + n.W2, n.h1, 0, 0, n.h1, dH1, n.h1, 0, H1, n.h1, 0, false);
    L.bwd_w(dH1, n.h1, 0, B, n.h1, mat(X, n.in), n.in, g + n.W1, n.in, 0, g + n.b1, 0);
}

// S[0..obs) = next_state of the record in physical slot `slot` (the newest transition of a rollout)
static __global__ void k_last_next_state(const uint32_t *__restrict__ records, prl_buf_layout L, int obs, int64_t slot, float *__restrict__ S) {
    const uint32_t *r = records + (size_t)slot * L.record_words;
    for (int p = threadIdx.x; p < obs; p += blockDim.x) S[p] = __uint_as_float(r[L.off_next_state + p]);
}

}  // namespace prl
