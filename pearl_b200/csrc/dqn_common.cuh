// dqn_common.cuh — definitions shared by the SIMT cooperative learner (dqn.cu) and the tensor-core
// one-SM-per-learner kernel (dqn_tc.cu).
#pragma once
#include "common.cuh"
#include "host_runtime.cuh"

namespace prl {

struct Dims {
    int obs, A, H1, H2, D, H1p, H2p, P, Pp;
    int oW1, ob1, oW2, ob2, oW3, ob3;
};

__host__ __device__ inline Dims make_dims(int obs, int A, int H1, int H2) {
    Dims d;
    d.obs = obs; d.A = A; d.H1 = H1; d.H2 = H2; d.D = obs + A;
    d.H1p = round_up(H1, 4); d.H2p = round_up(H2, 4);
    d.oW1 = 0; d.ob1 = d.oW1 + H1 * d.D; d.oW2 = d.ob1 + H1; d.ob2 = d.oW2 + H2 * H1;
    d.oW3 = d.ob2 + H2; d.ob3 = d.oW3 + H2; d.P = d.ob3 + 1;
    d.Pp = round_up(d.P + 1, 4);  // +1: the CTA's sum |q-y| rides along
    return d;
}


// soft target update, neural_networks/common/utils.py:214-226
__device__ __forceinline__ float soft_update(float src, float tgt, float tau, float omtau) {
    return __fadd_rn(__fmul_rn(tau, src), __fmul_rn(omtau, tgt));
}


// torch.optim.AdamW(amsgrad=True), non-capturable single-tensor path (torch/optim/adam.py:395-547):
// the scalars are evaluated on the host in double exactly as Python does and applied in fp32.
struct AdamScalars {
    float decay, omb1, beta2, omb2, eps, step_size, bc2_sqrt;
};
__device__ __forceinline__ float adamw_step(float *w, float *m_, float *v_, float *vmax_, float g, const AdamScalars &h) {
    float p = __fmul_rn(__ldcg(w), h.decay);                          // param.mul_(1 - lr*wd)
    float m = __ldcg(m_);
    m = fmaf(h.omb1, g - m, m);                                       // exp_avg.lerp_(grad, 1-beta1)
    float v = __fmul_rn(__ldcg(v_), h.beta2);
    v = __fadd_rn(v, __fmul_rn(__fmul_rn(h.omb2, g), g));             // .mul_(b2).addcmul_(g,g,1-b2)
    const float vm = fmaxf(__ldcg(vmax_), v);                         // amsgrad
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vm), h.bc2_sqrt), h.eps);
    p = __fadd_rn(p, __fdiv_rn(__fmul_rn(-h.step_size, m), denom));   // addcdiv_(m, denom, -step_size)
    *w = p; *m_ = m; *v_ = v; *vmax_ = vm;
    return p;
}

}  // namespace prl

struct prl_dqn {
    prl_dqn_cfg cfg;
    prl::Dims d;
    float *w, *wt, *m, *v, *vmax;
    int64_t adam_step;
    // workspace carve-up (device)
    float *gpart;
    int32_t *slots, *logical;
    float2 *scal_dev;
    uint32_t *tmp_rec;
    float *is_w, *td;         // prioritized replay: importance weights [rounds][B], |q-y| [B]
    void *multi_dev;          // 64 KB: per-learner descriptors of a multi-learner launch
    float *tc_tiles;          // operand-layout weight tiles of the tensor-core learner (dqn_tc.cu), or null
    int32_t *tmp_slots;
    prl_buf_layout tmp_lay;
    prl::Stage stage;         // pinned per-round optimizer scalars
    int sm_count, max_smem;
    int learn_smem, qv_smem;  // dynamic shared memory k_dqn_learn / k_q_values may use: max_smem minus their static part
    int last_launches, last_ctas, last_rows;
    // optional device timing of the persistent kernel (bench / roofline)
    int timing;
    cudaEvent_t t0, t1;
    long long *prof;
    prl_comm *comm;
};


int prl_dqn_stage_scalars(prl_dqn *q, int rounds, cudaStream_t stream);

// floats of the tensor-core learner's operand-layout weight tiles: per network W1 hi | W1 lo (64 x k1 each, k1 = obs
// rounded up to a multiple of 64) and W2 hi | W2 lo (64 x 64 each), online then target, and the online network's
// W2^T hi | W2^T lo (64 x 64 each); 0 for shapes outside its class
inline int64_t prl_tc_tile_floats(const prl_dqn_cfg *c) {
    if (c->hidden1 != 64 || c->hidden2 != 64 || c->obs_dim > 128 || c->obs_dim % 8) return 0;
    return 2ll * (128 * ((c->obs_dim + 63) & ~63) + 2 * 64 * 64) + 2 * 64 * 64;
}
