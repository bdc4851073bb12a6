// qrows.cuh — the per-row device code the discrete-action Q learners share (cql.cu, dueling.cu, multihead.cu, sarsa.cu,
// qrdqn.cu): the head of their per-call blocks, the loader of a warp's transition row, the warp's first argmax and the
// gradient of the reference's CQL term at the current slots.
#pragma once
#include <math.h>

#include "common.cuh"

namespace prl {

// the fields every Q learner's per-call block starts with
struct QCall {
    const int32_t *slots;                     // [rounds][B] (learn)
    float *out_loss;                          // [rounds]
    // learn_batch: the caller's dense batch
    const float *d_state, *d_next_state, *d_reward;
    const int32_t *d_action_id;
    const uint8_t *d_term;
    float decay;                              // AdamW decoupled decay 1 - lr * weight_decay
};

// ... and, where the next-action sets arrive compacted (available slots first), the caller's sets
struct QSetCall : QCall {
    const int32_t *d_next_ids, *d_next_cnt;   // [B][A] / [B]; may be null: every action available next
};

// the caller's available next-slot counts of a call block that has them; none: every slot counts
__device__ __forceinline__ const int32_t *next_counts(const QSetCall *c) { return c->d_next_cnt; }
__device__ __forceinline__ const int32_t *next_counts(const QCall *) { return nullptr; }

struct QRow {
    int action, cnt;                          // the taken action; the available next slots (kNext), clamped to A
    uint32_t flags;                           // the ring record's flags word (records != null)
};

// A warp's share of transition row w of a round: state and next state (lanes over the features), reward and terminated
// (lane 0) and, with kNext, the next-action id of every slot (lanes over the slots).  Returns the taken action and the
// available count (and the ring's flags word) to every lane.  records == null: the call block's dense batch, with its d_next_ids (null: slot k holds
// k) and next_counts (null: A); otherwise the record of the round's sampled slot, whose ids are its id bytes and its
// count bits 8..23 of the flags word when `dynamic`, every action otherwise.  The load kernels run it in blocks of 256
// threads under __launch_bounds__(256, 8): 32 registers, full occupancy.
template <bool kNext, class Call>
__device__ __forceinline__ QRow load_row(const uint32_t *__restrict__ records, const prl_buf_layout &L, int obs, int A, int dynamic,
                                         const Call *__restrict__ call, const int *__restrict__ round_idx, int B, int w, int lane,
                                         float *__restrict__ S,
                                         float *__restrict__ S2, float *__restrict__ R, float *__restrict__ T, int *__restrict__ ids) {
    QRow o;
    o.cnt = A;
    if (!records) {
        for (int p = lane; p < obs; p += 32) {
            S[(size_t)w * obs + p] = call->d_state[(size_t)w * obs + p];
            S2[(size_t)w * obs + p] = call->d_next_state[(size_t)w * obs + p];
        }
        if constexpr (kNext) {
            const int32_t *nid = call->d_next_ids, *ncnt = next_counts(call);
            for (int k = lane; k < A; k += 32) ids[(size_t)w * A + k] = nid ? nid[(size_t)w * A + k] : k;
            if (ncnt) o.cnt = min(ncnt[w], A);
        }
        o.action = call->d_action_id[w];
        if (lane == 0) {
            R[w] = call->d_reward[w];
            T[w] = call->d_term[w] ? 1.f : 0.f;
        }
        return o;
    }
    const uint32_t *r = records + (size_t)call->slots[(size_t)(*round_idx) * B + w] * L.record_words;
    for (int p = lane; p < obs; p += 32) {
        S[(size_t)w * obs + p] = __uint_as_float(r[L.off_state + p]);
        S2[(size_t)w * obs + p] = __uint_as_float(r[L.off_next_state + p]);
    }
    const uint32_t fl = r[L.off_flags];
    o.flags = fl;
    if constexpr (kNext) {
        const uint8_t *id8 = reinterpret_cast<const uint8_t *>(r + L.off_avail);
        for (int k = lane; k < A; k += 32) ids[(size_t)w * A + k] = dynamic ? (int)id8[k] : k;
        if (dynamic) o.cnt = min((int)((fl >> 8) & 0xffffu), A);
    }
    o.action = (int)r[L.off_action];
    if (lane == 0) {
        R[w] = __uint_as_float(r[L.off_reward]);
        T[w] = (fl & 1u) ? 1.f : 0.f;
    }
    return o;
}

// first argmax over a warp, ties to the lower slot (torch.argmax): each lane brings the best (value, slot) of its slots
__device__ __forceinline__ void warp_first_max(float &best, int &slot) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int ok = __shfl_xor_sync(0xffffffffu, slot, o);
        if (ov > best || (ov == best && ok < slot)) { best = ov; slot = ok; }
    }
}

// The gradient of alpha * the reference's CQL term (cql.cu) at the A current slots of a row, one warp:
//   d/dQ_k = alpha (softmax_k / B - n_k / (B A)),  n_0 = A - 1, n_1 = 1, n_k = 0 otherwise,
// with the logsumexp as a row max, then the sum of exp(l - max) (per lane in slot order, then a fixed tree).  value(k) is
// the online value of slot k; emit(k, g) takes the gradient of each of the lane's slots k = lane, lane + 32, ...
template <class Value, class Emit>
__device__ __forceinline__ void cql_slot_grad(int A, int B, float alpha, int lane, Value value, Emit emit) {
    float mx = -INFINITY;
    for (int k = lane; k < A; k += 32) mx = fmaxf(mx, value(k));
#pragma unroll
    for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float s = 0.f;
    for (int k = lane; k < A; k += 32) s += expf(value(k) - mx);
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float fB = (float)B, inv_ba = 1.f / ((float)B * (float)A);
    for (int k = lane; k < A; k += 32) {
        const float p = expf(value(k) - mx) / s;
        const float n_k = k == 0 ? (float)(A - 1) : (k == 1 ? 1.f : 0.f);
        emit(k, __fmul_rn(alpha, __fsub_rn(__fdiv_rn(p, fB), __fmul_rn(n_k, inv_ba))));
    }
}

}  // namespace prl
