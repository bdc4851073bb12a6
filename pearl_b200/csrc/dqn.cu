// dqn.cu — fused DQN / DoubleDQN learner: one persistent cooperative kernel runs
// `rounds` gradient steps (gather -> Q(s,a) -> Bellman target over all next
// actions -> MSE gradient -> backward -> AdamW(amsgrad) -> scheduled soft target
// update) without returning to the host.  See include/pearl_b200.h for the
// reference call sites each entry point replaces.
//
// Decomposition of one round over G CTAs (R = rows_per_cta batch rows each):
//   phase A (rows)   : each CTA evaluates its R transitions: online forward,
//                      target network on R*A (next_state, action) rows with the
//                      layer-1 state product shared across the A actions
//                      (one-hot action == one column of W1), backward, and
//                      writes its partial parameter gradient (fixed order).
//   grid barrier
//   phase B (update) : every thread owns a strided slice of the P parameters:
//                      sums the G partials in CTA order (deterministic),
//                      applies AdamW(amsgrad) and, when the NEXT round is a
//                      target-update round, the soft update.
//   grid barrier
// Parameters, Adam state and partials stay L2-resident; weights are streamed
// L2 -> shared panels (bypassing L1: they were written by other SMs).
#include <cooperative_groups.h>
#include <math.h>
#include <stdarg.h>

#include <new>

#include "common.cuh"
#include "sampler.cuh"
#include "dqn_common.cuh"

int prl_sampler_params(const prl_buf *b, int k, prl::SamplerParams *sp, size_t *smem_bytes);

namespace cg = cooperative_groups;
using namespace prl;

namespace {

constexpr int NT = 256;      // threads per CTA
constexpr int NC = 64;       // output columns per staged weight panel
constexpr int KCMAX = 128;   // K extent of a staged weight panel
constexpr int MB = 64;       // rows per register-tiled row block
constexpr int STAGE_FLOATS = KCMAX * (NC + 4);  // >= NC * (KCMAX + 4): either panel orientation
constexpr int RED_FLOATS = NT * 16;

// shared-memory plan, offsets in floats (all multiples of 4)
struct Plan {
    int rec, T1o, H1o, H2o, T1t, T1d, dZ2, dZ1, Hc, H2c, WaO, WaT, qa, scal, stage, red, own, total;
    int zero_begin, zero_end;  // activation region zero-initialised once
};

__host__ __device__ inline Plan make_plan(const Dims &d, int R, int W, int mch) {
    Plan p;
    int o = 0;
    p.rec = o; o += 2 * R * W;
    p.zero_begin = o;
    p.T1o = o; o += R * d.H1p;
    p.H1o = o; o += R * d.H1p;
    p.H2o = o; o += R * d.H2p;
    p.T1t = o; o += R * d.H1p;
    p.T1d = o; o += R * d.H1p;
    p.dZ2 = o; o += R * d.H2p;
    p.dZ1 = o; o += R * d.H1p;
    p.Hc = o; o += mch * d.H1p;
    p.H2c = o; o += mch * d.H2p;
    p.WaO = o; o += d.A * d.H1p;
    p.WaT = o; o += d.A * d.H1p;
    p.qa = o; o += round_up(R * d.A, 4);
    p.scal = o; o += round_up(9 * R, 4);
    p.zero_end = o;
    p.stage = o; o += STAGE_FLOATS;
    p.red = o; o += RED_FLOATS;
    p.own = o; o += round_up(2 * (R + 1) + 16, 4);   // sharded replay: per round parity [count, batch index of each owned row], scan scratch
    p.total = o;
    return p;
}

struct LearnArgs {
    const uint32_t *records;
    prl_buf_layout lay;
    int buf_flags;
    const int32_t *slots;     // [rounds][B] physical record index
    float *w, *wt, *m, *v, *vmax;
    float *gpart;             // [G][Pp]
    const float2 *scal;       // [rounds] (step_size, sqrt(bias_correction2)) as torch computes them
    float *out_mae, *out_q, *out_y;
    const float *is_weight;   // optional [rounds][B] importance weights (prioritized replay)
    float *out_td;            // optional [rounds][B] |q - y| per row
    Dims d;
    Plan plan;
    int B, R, rounds, mch, double_dqn, freq;
    int first_update;         // apply the soft target update before round 0
    int G;                    // learner CTAs; CTA index G (if fused_sampler) produces the indices
    int fused_sampler;
    SamplerParams sp;         // out_slot == slots (+ optional out_logical)
    uint32_t *mt_state;
    // data-parallel exchange (world == 1: unused)
    int rank, world;
    float *peer_inbox[16];
    unsigned int *peer_flags[16];
    float *inbox;             // local inbox [2][world][comm_slot]
    unsigned int *flags;      // local arrival counters, one per learner CTA
    long long comm_slot;      // floats per inbox slot
    unsigned long long exch0; // exchanges completed before this launch
    float inv_world;
    // replay sharded over the ranks (SURVEY.md 8e): every rank draws the SAME B global indices; transition number g
    // (global write counter) lives on rank g mod W at local slot (g div W) mod local_cap; a rank works on the rows it owns
    int shard_world, shard_rank;
    long long g_oldest, local_cap;
    long long *prof;          // optional [rounds][16] SM-clock stamps of CTA 0 (developer profiling)
    long long steps0;         // learner._training_steps before the call
    float decay, omb1, beta2, omb2, eps, gamma, tau, omtau, inv_b2;  // fp32 images of the scalars
};

// ---------------------------------------------------------------------------
// out[m][n] = act(bias[n] + sum_k X[m][k] * Wop[n][k]),  m < M, n < N, k < K
//   X   : shared, row stride ldx (multiple of 4, rows 16-byte aligned)
//   Wop : global.  NN == false: Wop[n][k] = W[n*ldw + k]  (y = x W^T, forward)
//                  NN == true : Wop[n][k] = W[k*ldw + n]  (y = x W,   backward wrt input)
//   out : shared, row stride ldo
// The weight panel (<= 64 outputs x <= 128 k) is streamed L2 -> shared with
// 16-byte cp.async (all chunks in flight at once; zero-filled tails), then
// consumed by 4x4 register tiles.  Row blocks with few rows let the idle thread
// rows split K; the partial sums are combined in fixed order through `red`.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16_zfill(void *smem_dst, const void *gmem_src, int src_bytes) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem_src), "r"(src_bytes)
                 : "memory");
}

template <bool NN>
__device__ __noinline__ void cta_linear(const float *X, int ldx, int M, const float *__restrict__ W, int ldw, int N, int K,
                           const float *__restrict__ bias, bool relu, float *out, int ldo, float *stage,
                           float *red) {
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(W) & 15) == 0) && ((ldw & 3) == 0);
    for (int n0 = 0; n0 < N; n0 += NC) {
        const int nc = min(NC, N - n0);
        for (int m0 = 0; m0 < M; m0 += MB) {
            const int mb = min(MB, M - m0);
            const int mt_cnt = (mb + 3) >> 2;
            int mtp = 1, sh = 0;
            while (mtp < mt_cnt) { mtp <<= 1; sh++; }
            const int KS = 16 >> sh;
            const int mt = ty & (mtp - 1), kz = ty >> sh;
            const bool active = mt < mt_cnt;
            float acc[4][4];
#pragma unroll
            for (int i = 0; i < 4; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
            const float *xr[4];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                int m = m0 + mt * 4 + i;
                if (m > M - 1) m = M - 1;
                xr[i] = X + (size_t)m * ldx;
            }
            for (int k0 = 0; k0 < K; k0 += KCMAX) {
                const int kc = min(KCMAX, K - k0);
                const int kc4 = round_up(kc, 4);
                // panel geometry: NT rows = outputs, cols = k; NN rows = k, cols = outputs
                const int prow = NN ? kc4 : NC, pcol = NN ? NC : kc4;
                const int vrow = NN ? kc : nc, vcol = NN ? nc : kc;       // valid extent
                const int lds = NN ? (NC + 4) : (kc4 | 4);                // (lds/4) odd
                const float *src = NN ? (W + (size_t)k0 * ldw + n0) : (W + (size_t)n0 * ldw + k0);
                __syncthreads();  // previous panel fully consumed
                if (vec_ok) {
                    const int c4 = pcol >> 2;
                    for (int e = tid; e < prow * c4; e += NT) {
                        const int r = e / c4, c = (e - r * c4) * 4;
                        int nb = 0;
                        if (r < vrow) nb = 4 * max(0, min(4, vcol - c));
                        cp_async16_zfill(stage + r * lds + c, nb ? (src + (size_t)r * ldw + c) : W, nb);
                    }
                    cp_async_commit();
                    cp_async_wait<0>();
                } else {  // unaligned parameter block: scalar loads, 8 in flight per thread
                    const int tr = tid / pcol, tc = tid - tr * pcol, rpp = NT / pcol;
                    if (tr < rpp)
                        for (int r = tr; r < prow; r += rpp * 8) {
                            float v[8];
#pragma unroll
                            for (int u = 0; u < 8; u++) {
                                const int rr = r + u * rpp;
                                v[u] = (rr < vrow && tc < vcol) ? __ldcg(src + (size_t)rr * ldw + tc) : 0.f;
                            }
#pragma unroll
                            for (int u = 0; u < 8; u++) {
                                const int rr = r + u * rpp;
                                if (rr < prow) stage[rr * lds + tc] = v[u];
                            }
                        }
                }
                __syncthreads();
                if (active) {
                    const int ksl = round_up((kc4 + KS - 1) / KS, 4);
                    const int kb = kz * ksl, ke = min(kc4, kb + ksl);
                    if (!NN) {
                        for (int k = kb; k < ke; k += 4) {
                            float4 a[4], b[4];
#pragma unroll
                            for (int i = 0; i < 4; i++) a[i] = *reinterpret_cast<const float4 *>(xr[i] + k0 + k);
#pragma unroll
                            for (int j = 0; j < 4; j++)
                                b[j] = *reinterpret_cast<const float4 *>(stage + (tx + 16 * j) * lds + k);
#pragma unroll
                            for (int i = 0; i < 4; i++)
#pragma unroll
                                for (int j = 0; j < 4; j++) {
                                    acc[i][j] = fmaf(a[i].x, b[j].x, acc[i][j]);
                                    acc[i][j] = fmaf(a[i].y, b[j].y, acc[i][j]);
                                    acc[i][j] = fmaf(a[i].z, b[j].z, acc[i][j]);
                                    acc[i][j] = fmaf(a[i].w, b[j].w, acc[i][j]);
                                }
                        }
                    } else {
                        for (int k = kb; k < ke; k += 4) {
                            float4 a[4];
#pragma unroll
                            for (int i = 0; i < 4; i++) a[i] = *reinterpret_cast<const float4 *>(xr[i] + k0 + k);
#pragma unroll
                            for (int kk = 0; kk < 4; kk++) {
                                const float4 b = *reinterpret_cast<const float4 *>(stage + (k + kk) * lds + tx * 4);
#pragma unroll
                                for (int i = 0; i < 4; i++) {
                                    const float av = kk == 0 ? a[i].x : kk == 1 ? a[i].y : kk == 2 ? a[i].z : a[i].w;
                                    acc[i][0] = fmaf(av, b.x, acc[i][0]);
                                    acc[i][1] = fmaf(av, b.y, acc[i][1]);
                                    acc[i][2] = fmaf(av, b.z, acc[i][2]);
                                    acc[i][3] = fmaf(av, b.w, acc[i][3]);
                                }
                            }
                        }
                    }
                }
            }
            if (KS > 1) {
                // combine the K slices in fixed order kz = 0,1,2,...: every thread reduces and
                // finishes a strided share of the block's outputs (not just the kz == 0 threads)
                __syncthreads();
#pragma unroll
                for (int e = 0; e < 16; e++) red[(ty * 16 + e) * 16 + tx] = acc[e >> 2][e & 3];
                __syncthreads();
                const int n_out = mt_cnt * 256;  // (mt, e, tx)
                for (int o = tid; o < n_out; o += NT) {
                    const int otx = o & 15, oe = (o >> 4) & 15, omt = o >> 8;
                    float v = 0.f;
                    for (int z = 0; z < KS; z++) v += red[(((z << sh) + omt) * 16 + oe) * 16 + otx];
                    const int m = m0 + omt * 4 + (oe >> 2);
                    const int n = n0 + (NN ? otx * 4 + (oe & 3) : otx + 16 * (oe & 3));
                    if (m < M && n < N) {
                        if (bias) v += __ldcg(bias + n);
                        if (relu) v = fmaxf(v, 0.f);
                        out[(size_t)m * ldo + n] = v;
                    }
                }
            } else if (active) {
                float bv[4];
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const int n = n0 + (NN ? tx * 4 + j : tx + 16 * j);
                    bv[j] = (bias && n < N) ? __ldcg(bias + n) : 0.f;
                }
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const int m = m0 + mt * 4 + i;
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        const int n = n0 + (NN ? tx * 4 + j : tx + 16 * j);
                        float v = acc[i][j] + bv[j];
                        if (relu) v = fmaxf(v, 0.f);
                        if (m < M && n < N) out[(size_t)m * ldo + n] = v;
                    }
                }
            }
        }
    }
    __syncthreads();
}

// out[n*ldw + k] = sum_{m<M} dY[m][n] * X[m][k]  (n < N, k < K): the CTA's partial
// weight gradient, written to global in the parameter layout.
__device__ __noinline__ void cta_outer(const float *dY, int ldy, const float *X, int ldx, int M, int N, int K,
                          float *__restrict__ out, int ldw) {
    const int K4 = (K + 3) >> 2;
    for (int item = threadIdx.x; item < N * K4; item += NT) {
        const int n = item / K4, k = (item - n * K4) * 4;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int m = 0; m < M; m++) {
            const float dy = dY[m * ldy + n];
            const float4 x = *reinterpret_cast<const float4 *>(X + (size_t)m * ldx + k);
            acc.x = fmaf(dy, x.x, acc.x); acc.y = fmaf(dy, x.y, acc.y);
            acc.z = fmaf(dy, x.z, acc.z); acc.w = fmaf(dy, x.w, acc.w);
        }
        float *o = out + (size_t)n * ldw + k;
        if (k + 3 < K && ((reinterpret_cast<uintptr_t>(o) & 15) == 0)) {
            *reinterpret_cast<float4 *>(o) = acc;
        } else {
            o[0] = acc.x;
            if (k + 1 < K) o[1] = acc.y;
            if (k + 2 < K) o[2] = acc.z;
            if (k + 3 < K) o[3] = acc.w;
        }
    }
}

// q[m] = b3 + sum_j w3[j] * H[m][j]   (one warp per row, fixed shuffle tree)
__device__ __noinline__ void cta_head(const float *H, int ldh, int M, const float *__restrict__ w3, float b3, int H2,
                         float *q) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float wv[8];  // this lane's slice of w3, fetched from L2 once (covers H2 <= 256 without reloads)
#pragma unroll
    for (int u = 0; u < 8; u++) wv[u] = (lane + 32 * u < H2) ? __ldcg(w3 + lane + 32 * u) : 0.f;
    for (int m = warp; m < M; m += NT / 32) {
        float s = 0.f;
#pragma unroll
        for (int u = 0; u < 8; u++)
            if (lane + 32 * u < H2) s = fmaf(wv[u], H[(size_t)m * ldh + lane + 32 * u], s);
        for (int j = lane + 256; j < H2; j += 32) s = fmaf(__ldcg(w3 + j), H[(size_t)m * ldh + j], s);
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) q[m] = s + b3;
    }
}

// action columns of W1 transposed into shared: WaT[a][j] = W1[j][obs + a]
__device__ __noinline__ void stage_action_cols(const float *__restrict__ w, const Dims &d, float *Wa) {
    for (int e = threadIdx.x; e < d.A * d.H1; e += NT) {
        const int j = e / d.A, a = e - j * d.A;
        Wa[a * d.H1p + j] = __ldcg(w + d.oW1 + (size_t)j * d.D + d.obs + a);
    }
}

struct RowScal {  // views into the per-row scalar block
    int *act, *cnt, *idsel;
    float *rew, *term, *q, *y, *dq, *v;
};
__device__ inline RowScal row_scal(float *base, int R) {
    RowScal s;
    s.act = reinterpret_cast<int *>(base);
    s.cnt = reinterpret_cast<int *>(base + R);
    s.idsel = reinterpret_cast<int *>(base + 2 * R);
    s.rew = base + 3 * R; s.term = base + 4 * R; s.q = base + 5 * R;
    s.y = base + 6 * R; s.dq = base + 7 * R; s.v = base + 8 * R;
    return s;
}

// Q(s', a) for every (row, available-action slot): qa[r*A + a]; -inf where masked.
// T1 = layer-1 state product (+bias) of the net being evaluated, Wa its action columns.
__device__ __noinline__ void all_actions_q(const float *__restrict__ net, const Dims &d, const float *T1, const float *Wa,
                              const uint32_t *rec, int W, const prl_buf_layout &L, int buf_flags, int Rv,
                              int mch, const int *cnt, float *Hc, float *H2c, float *qa, float *stage,
                              float *red) {
    const int MA = Rv * d.A;
    for (int c0 = 0; c0 < MA; c0 += mch) {
        const int mc = min(mch, MA - c0);
        for (int e = threadIdx.x; e < mc * d.H1; e += NT) {
            const int ra = e / d.H1, j = e - ra * d.H1;
            const int r = (c0 + ra) / d.A, a = (c0 + ra) - r * d.A;
            int id = a;
            if (buf_flags & PRL_BUF_DYNAMIC_ACTIONS)
                id = reinterpret_cast<const uint8_t *>(rec + (size_t)r * W + L.off_avail)[a];
            Hc[ra * d.H1p + j] = fmaxf(T1[r * d.H1p + j] + Wa[id * d.H1p + j], 0.f);
        }
        __syncthreads();
        cta_linear<false>(Hc, d.H1p, mc, net + d.oW2, d.H1, d.H2, d.H1, net + d.ob2, true, H2c, d.H2p, stage, red);
        cta_head(H2c, d.H2p, mc, net + d.oW3, __ldcg(net + d.ob3), d.H2, qa + c0);
        __syncthreads();
    }
    for (int e = threadIdx.x; e < MA; e += NT) {
        const int r = e / d.A, a = e - r * d.A;
        if (a >= cnt[r]) qa[e] = -INFINITY;  // next_state_action_values[mask] = -inf
    }
    __syncthreads();
}

// rows of `round` this CTA works on: r0 .. r0 + Rv - 1 of the batch, or — sharded replay — the owned rows whose
// position k in the rank's compacted list has k mod G == blockIdx.x
__device__ int prefetch_records(const LearnArgs &a, float *sm, int round, int Rv, int r0) {
    const int W = a.lay.record_words, W4 = W >> 2;
    uint32_t *dst = reinterpret_cast<uint32_t *>(sm + a.plan.rec) + (size_t)(round & 1) * a.R * W;
    const int32_t *sl = a.slots + (size_t)round * a.B;
    if (a.shard_world > 1) {
        int *own = reinterpret_cast<int *>(sm + a.plan.own) + (round & 1) * (a.R + 1);
        int *wsum = reinterpret_cast<int *>(sm + a.plan.own) + 2 * (a.R + 1);
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        int base = 0;
        for (int i0 = 0; i0 < a.B; i0 += NT) {
            const int i = i0 + threadIdx.x;
            bool mine = false;
            if (i < a.B) mine = (int)((a.g_oldest + (long long)__ldcg(sl + i)) % a.shard_world) == a.shard_rank;
            const unsigned bal = __ballot_sync(0xffffffffu, mine);
            if (lane == 0) wsum[warp] = __popc(bal);
            __syncthreads();
            int off = base, total = 0;
            for (int w8 = 0; w8 < NT / 32; w8++) { if (w8 < warp) off += wsum[w8]; total += wsum[w8]; }
            const int k = off + __popc(bal & ((1u << lane) - 1u));
            if (mine && k % a.G == (int)blockIdx.x) own[1 + k / a.G] = i;
            base += total;
            __syncthreads();
        }
        Rv = base > (int)blockIdx.x ? (base - (int)blockIdx.x + a.G - 1) / a.G : 0;
        if (threadIdx.x == 0) own[0] = Rv;
        __syncthreads();
        for (int e = threadIdx.x; e < Rv * W4; e += NT) {
            const int r = e / W4, c = e - r * W4;
            const long long g = a.g_oldest + (long long)__ldcg(sl + own[1 + r]);
            const long long slot = (g / a.shard_world) % a.local_cap;
            cp_async16(dst + (size_t)r * W + c * 4, a.records + (size_t)slot * W + c * 4);
        }
        cp_async_commit();
        return Rv;
    }
    sl += r0;
    for (int e = threadIdx.x; e < Rv * W4; e += NT) {
        const int r = e / W4, c = e - r * W4;
        cp_async16(dst + (size_t)r * W + c * 4, a.records + (size_t)__ldcg(sl + r) * W + c * 4);
    }
    cp_async_commit();
    return Rv;
}

// ---------------------------------------------------------------------------
// phase A
// ---------------------------------------------------------------------------
#define PRL_STAMP(idx)                                                                  \
    do {                                                                                \
        if (a.prof && blockIdx.x == 0 && threadIdx.x == 0) a.prof[(size_t)round * 16 + (idx)] = clock64(); \
    } while (0)

__device__ void phase_rows(const LearnArgs &a, float *sm, int round) {
    const Dims &d = a.d;
    const Plan &pl = a.plan;
    const int tid = threadIdx.x, R = a.R, W = a.lay.record_words;
    const int r0 = blockIdx.x * R;
    int Rv = min(R, a.B - r0);
    const int *own = reinterpret_cast<const int *>(sm + pl.own) + (round & 1) * (R + 1);
    const bool shard = a.shard_world > 1;
    if (shard) Rv = own[0];                       // written (and barrier-published) by prefetch_records of this round
    PRL_STAMP(0);
    cp_async_wait<0>();
    __syncthreads();
    PRL_STAMP(1);

    const uint32_t *rec = reinterpret_cast<const uint32_t *>(sm + pl.rec) + (size_t)(round & 1) * R * W;
    const float *recf = reinterpret_cast<const float *>(rec);
    RowScal sc = row_scal(sm + pl.scal, R);
    float *stage = sm + pl.stage, *red = sm + pl.red;
    float *T1o = sm + pl.T1o, *H1o = sm + pl.H1o, *H2o = sm + pl.H2o, *T1t = sm + pl.T1t, *T1d = sm + pl.T1d;
    float *dZ2 = sm + pl.dZ2, *dZ1 = sm + pl.dZ1, *Hc = sm + pl.Hc, *H2c = sm + pl.H2c;
    float *WaO = sm + pl.WaO, *WaT = sm + pl.WaT, *qa = sm + pl.qa;
    const float *w = a.w, *wt = a.wt;

    if (tid < Rv) {
        const uint32_t *r = rec + (size_t)tid * W;
        sc.act[tid] = (int)r[a.lay.off_action];
        sc.rew[tid] = __uint_as_float(r[a.lay.off_reward]);
        const uint32_t fl = r[a.lay.off_flags];
        sc.term[tid] = (fl & 1u) ? 1.f : 0.f;
        sc.cnt[tid] = (int)((fl >> 8) & 0xffffu);
    }
    stage_action_cols(w, d, WaO);
    stage_action_cols(wt, d, WaT);
    __syncthreads();
    PRL_STAMP(2);

    // ---- online Q(s, a) (q_value_networks.py:152-174; the one-hot action selects a W1 column)
    cta_linear<false>(recf + a.lay.off_state, W, Rv, w + d.oW1, d.D, d.H1, d.obs, w + d.ob1, false, T1o, d.H1p,
                      stage, red);
    for (int e = tid; e < Rv * d.H1; e += NT) {
        const int r = e / d.H1, j = e - r * d.H1;
        H1o[r * d.H1p + j] = fmaxf(T1o[r * d.H1p + j] + WaO[sc.act[r] * d.H1p + j], 0.f);
    }
    __syncthreads();
    PRL_STAMP(3);
    cta_linear<false>(H1o, d.H1p, Rv, w + d.oW2, d.H1, d.H2, d.H1, w + d.ob2, true, H2o, d.H2p, stage, red);
    cta_head(H2o, d.H2p, Rv, w + d.oW3, __ldcg(w + d.ob3), d.H2, sc.q);
    PRL_STAMP(4);

    // ---- bootstrap value of s' (deep_q_learning.py:130-167 / double_dqn.py:29-57)
    cta_linear<false>(recf + a.lay.off_next_state, W, Rv, wt + d.oW1, d.D, d.H1, d.obs, wt + d.ob1, false, T1t,
                      d.H1p, stage, red);
    PRL_STAMP(5);
    if (!a.double_dqn) {
        all_actions_q(wt, d, T1t, WaT, rec, W, a.lay, a.buf_flags, Rv, a.mch, sc.cnt, Hc, H2c, qa, stage, red);
        if (tid < Rv) {
            float best = -INFINITY;
            for (int k = 0; k < d.A; k++) best = fmaxf(best, qa[tid * d.A + k]);
            sc.v[tid] = best;
        }
    } else {
        cta_linear<false>(recf + a.lay.off_next_state, W, Rv, w + d.oW1, d.D, d.H1, d.obs, w + d.ob1, false, T1d,
                          d.H1p, stage, red);
        all_actions_q(w, d, T1d, WaO, rec, W, a.lay, a.buf_flags, Rv, a.mch, sc.cnt, Hc, H2c, qa, stage, red);
        if (tid < Rv) {
            float best = qa[tid * d.A];
            int arg = 0;
            for (int k = 1; k < d.A; k++) {
                const float x = qa[tid * d.A + k];
                if (x > best) { best = x; arg = k; }
            }
            int id = arg;  // padded slots hold action id 0 (tensor_based_replay_buffer.py:228-236)
            if (arg >= sc.cnt[tid]) id = 0;
            else if (a.buf_flags & PRL_BUF_DYNAMIC_ACTIONS)
                id = reinterpret_cast<const uint8_t *>(rec + (size_t)tid * W + a.lay.off_avail)[arg];
            sc.idsel[tid] = id;
        }
        __syncthreads();
        for (int e = tid; e < Rv * d.H1; e += NT) {
            const int r = e / d.H1, j = e - r * d.H1;
            Hc[r * d.H1p + j] = fmaxf(T1t[r * d.H1p + j] + WaT[sc.idsel[r] * d.H1p + j], 0.f);
        }
        __syncthreads();
        cta_linear<false>(Hc, d.H1p, Rv, wt + d.oW2, d.H1, d.H2, d.H1, wt + d.ob2, true, H2c, d.H2p, stage, red);
        cta_head(H2c, d.H2p, Rv, wt + d.oW3, __ldcg(wt + d.ob3), d.H2, sc.v);
    }
    __syncthreads();

    PRL_STAMP(6);
    // ---- Bellman target, MSE gradient (deep_td_learning.py:313-320)
    if (tid < Rv) {
        const float y = __fadd_rn(__fmul_rn(__fmul_rn(sc.v[tid], a.gamma), 1.f - sc.term[tid]), sc.rew[tid]);
        const float q = sc.q[tid];
        sc.y[tid] = y;
        float dqv = (q - y) * a.inv_b2;  // d/dq mean((q-y)^2) = 2 (q-y) / B
        const int bi = shard ? own[1 + tid] : r0 + tid;   // position of this row in the sampled batch
        if (a.is_weight) dqv *= __ldg(a.is_weight + (size_t)round * a.B + bi);   // d/dq mean(w (q-y)^2)
        sc.dq[tid] = dqv;
        if (a.out_td) a.out_td[(size_t)round * a.B + bi] = fabsf(q - y);
        if (a.out_q) a.out_q[(size_t)round * a.B + bi] = q;
        if (a.out_y) a.out_y[(size_t)round * a.B + bi] = y;
    }
    __syncthreads();

    PRL_STAMP(7);
    // ---- backward through the online network
    for (int e = tid; e < Rv * d.H2; e += NT) {
        const int r = e / d.H2, j = e - r * d.H2;
        dZ2[r * d.H2p + j] = (H2o[r * d.H2p + j] > 0.f) ? sc.dq[r] * __ldcg(w + d.oW3 + j) : 0.f;
    }
    __syncthreads();
    cta_linear<true>(dZ2, d.H2p, Rv, w + d.oW2, d.H1, d.H1, d.H2, nullptr, false, dZ1, d.H1p, stage, red);
    for (int e = tid; e < Rv * d.H1; e += NT) {
        const int r = e / d.H1, j = e - r * d.H1;
        if (!(H1o[r * d.H1p + j] > 0.f)) dZ1[r * d.H1p + j] = 0.f;
    }
    __syncthreads();

    PRL_STAMP(8);
    // next round's transitions: issued after the last weight panel (cp.async groups retire
    // in order) so the HBM latency hides behind the outer products, phase B and the barriers
    if (round + 1 < a.rounds) prefetch_records(a, sm, round + 1, Rv, r0);
    PRL_STAMP(13);
    float *g = a.gpart + (size_t)blockIdx.x * d.Pp;
    cta_outer(dZ1, d.H1p, recf + a.lay.off_state, W, Rv, d.H1, d.obs, g + d.oW1, d.D);  // dW1[:, :obs]
    cta_outer(dZ2, d.H2p, H1o, d.H1p, Rv, d.H2, d.H1, g + d.oW2, d.H1);                 // dW2
    PRL_STAMP(14);
    for (int e = tid; e < d.H1 * d.A; e += NT) {                                        // dW1[:, obs+a]
        const int j = e / d.A, k = e - j * d.A;
        float s = 0.f;
        for (int r = 0; r < Rv; r++)
            if (sc.act[r] == k) s += dZ1[r * d.H1p + j];
        g[d.oW1 + (size_t)j * d.D + d.obs + k] = s;
    }
    PRL_STAMP(15);
    for (int j = tid; j < d.H1; j += NT) {
        float s = 0.f;
        for (int r = 0; r < Rv; r++) s += dZ1[r * d.H1p + j];
        g[d.ob1 + j] = s;
    }
    for (int j = tid; j < d.H2; j += NT) {
        float s = 0.f, s3 = 0.f;
        for (int r = 0; r < Rv; r++) {
            s += dZ2[r * d.H2p + j];
            s3 = fmaf(sc.dq[r], H2o[r * d.H2p + j], s3);
        }
        g[d.ob2 + j] = s;
        g[d.oW3 + j] = s3;
    }
    if (tid == 0) {
        float s = 0.f, e = 0.f;
        for (int r = 0; r < Rv; r++) { s += sc.dq[r]; e += fabsf(sc.q[r] - sc.y[r]); }
        g[d.ob3] = s;
        g[d.P] = e;
    }
    PRL_STAMP(9);
}

// ---------------------------------------------------------------------------
// phase B: gradient reduction + AdamW(amsgrad) (torch/optim/adam.py:395-547,
// non-capturable single-tensor path) + look-ahead soft target update
// ---------------------------------------------------------------------------
__device__ __forceinline__ void st_volatile_v2(float *p, float val, unsigned int tag) {
    asm volatile("st.volatile.global.v2.b32 [%0], {%1, %2};" ::"l"(p), "r"(__float_as_uint(val)), "r"(tag) : "memory");
}
__device__ __forceinline__ void ld_volatile_v2(const float *p, float &val, unsigned int &tag) {
    unsigned int a, b;
    asm volatile("ld.volatile.global.v2.b32 {%0, %1}, [%2];" : "=r"(a), "=r"(b) : "l"(p) : "memory");
    val = __uint_as_float(a);
    tag = b;
}

// sum of the G partials of parameter i in CTA order; up to 32 loads in flight
__device__ __forceinline__ float reduce_partials(const LearnArgs &a, int i) {
    const Dims &d = a.d;
    const int G = a.G;
    float g = 0.f;
    int c = 0;
    for (; c + 32 <= G; c += 32) {
        float t[32];
#pragma unroll
        for (int u = 0; u < 32; u++) t[u] = __ldcg(a.gpart + (size_t)(c + u) * d.Pp + i);
#pragma unroll
        for (int u = 0; u < 32; u++) g += t[u];
    }
    for (; c + 8 <= G; c += 8) {
        float t[8];
#pragma unroll
        for (int u = 0; u < 8; u++) t[u] = __ldcg(a.gpart + (size_t)(c + u) * d.Pp + i);
#pragma unroll
        for (int u = 0; u < 8; u++) g += t[u];
    }
    for (; c < G; c++) g += __ldcg(a.gpart + (size_t)c * d.Pp + i);
    return g;
}

__device__ void phase_update(const LearnArgs &a, int round) {
    const Dims &d = a.d;
    const int G = a.G;
    const float2 s = a.scal[round];
    const float step_size = s.x, bc2_sqrt = s.y;
    const long long t_next = a.steps0 + round + 2;  // training step of the next round
    const bool upd_next = (round + 1 < a.rounds) && ((t_next + 1) % a.freq == 0);
    const int parity = (int)((a.exch0 + (unsigned long long)round) & 1ull);
    const unsigned int seq = (unsigned int)(a.exch0 + (unsigned long long)round + 1ull);
    const int nx = d.P + (a.shard_world > 1 ? 1 : 0);   // sharded replay: sum |q - y| travels with the gradient
    if (a.world > 1) {
        // ---- fused gradient exchange (NVLink peer memory, one-way latency only): every rank
        // pushes (value, round sequence number) as ONE 8-byte store into every peer's inbox;
        // readers poll the sequence half of each element, so there is no fence / flag round trip.
        for (int i = blockIdx.x * NT + threadIdx.x; i < nx; i += G * NT) {
            const float g = reduce_partials(a, i);
            const size_t off = ((size_t)parity * a.world + a.rank) * a.comm_slot + i;
            for (int p = 0; p < a.world; p++) st_volatile_v2(a.peer_inbox[p] + 2 * off, g, seq);
        }
    }
    for (int i = blockIdx.x * NT + threadIdx.x; i <= d.P; i += G * NT) {
        float g;
        if (a.world > 1 && i < nx) {
            float sum = 0.f;  // rank order: identical on every rank
            for (int q = 0; q < a.world; q++) {
                const float *src = a.inbox + 2 * (((size_t)parity * a.world + q) * a.comm_slot + i);
                float val;
                unsigned int tag;
                do { ld_volatile_v2(src, val, tag); } while (tag != seq);
                sum += val;
            }
            g = sum * a.inv_world;
        } else {
            g = reduce_partials(a, i);
        }
        if (i == d.P) {  // reported "loss": mean |q - y| (deep_td_learning.py:358-360), local batch
            a.out_mae[round] = g / (float)a.B;
            continue;
        }
        AdamScalars hs{a.decay, a.omb1, a.beta2, a.omb2, a.eps, step_size, bc2_sqrt};
        const float p = adamw_step(a.w + i, a.m + i, a.v + i, a.vmax + i, g, hs);
        if (upd_next) a.wt[i] = soft_update(p, __ldcg(a.wt + i), a.tau, a.omtau);
    }
}

__global__ void __launch_bounds__(NT, 1) k_dqn_learn(const LearnArgs a) {
    extern __shared__ __align__(16) float sm[];
    cg::grid_group grid = cg::this_grid();
    if (a.fused_sampler && blockIdx.x == a.G) {
        // ---- producer CTA: the MT19937-exact index stream, two rounds ahead of the learners,
        // fully overlapped with their work; it only meets them at the grid barriers.
        __shared__ SamplerState S;
        sampler_init(S, a.mt_state, sm, a.sp);
        sampler_advance(S, sm, a.sp, min(a.rounds, 2));
        __threadfence();
        grid.sync();
        if (a.first_update) grid.sync();
        for (int round = 0; round < a.rounds; round++) {
            sampler_advance(S, sm, a.sp, min(a.rounds, round + 3));
            __threadfence();
            grid.sync();
            grid.sync();
        }
        __syncthreads();
        sampler_store(S, a.mt_state);
        return;
    }
    const int r0 = blockIdx.x * a.R, Rv = min(a.R, a.B - r0);
    for (int i = a.plan.zero_begin + threadIdx.x; i < a.plan.zero_end; i += NT) sm[i] = 0.f;
    if (a.fused_sampler) grid.sync();  // indices of rounds 0 and 1 are published
    prefetch_records(a, sm, 0, Rv, r0);
    // forward() applies the soft update BEFORE the gradient step of a round with
    // (training_steps + 1) % freq == 0 (deep_td_learning.py:283-284); later rounds get
    // it from phase B of the previous round.
    if (a.first_update) {
        for (int i = blockIdx.x * NT + threadIdx.x; i < a.d.P; i += a.G * NT)
            a.wt[i] = soft_update(__ldcg(a.w + i), __ldcg(a.wt + i), a.tau, a.omtau);
        __threadfence();
        grid.sync();
    }
    for (int round = 0; round < a.rounds; round++) {
        phase_rows(a, sm, round);
        __threadfence();
        grid.sync();
        PRL_STAMP(10);
        phase_update(a, round);
        PRL_STAMP(11);
        __threadfence();
        grid.sync();
        PRL_STAMP(12);
    }
    cp_async_wait<0>();
}

// ---------------------------------------------------------------------------
// learn_batch support: pack a caller-supplied TransitionBatch into records
// (always with explicit next-action lists; an arbitrary mask is compacted to a
// prefix, which leaves max / first-argmax over the available set unchanged)
// ---------------------------------------------------------------------------
__global__ void k_pack_batch(uint32_t *__restrict__ rec, prl_buf_layout L, int obs, int A, int n,
                             const float *__restrict__ state, const long long *__restrict__ action,
                             const float *__restrict__ reward, const float *__restrict__ next_state,
                             const uint8_t *__restrict__ terminated, const float *__restrict__ next_avail,
                             const uint8_t *__restrict__ mask, int32_t *__restrict__ slots) {
    const int lane = threadIdx.x & 31;
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (w >= n) return;
    uint32_t *r = rec + (size_t)w * L.record_words;
    for (int p = lane; p < L.record_words; p += 32) r[p] = 0;
    __syncwarp();
    for (int p = lane; p < obs; p += 32) {
        r[L.off_state + p] = __float_as_uint(state[(size_t)w * obs + p]);
        r[L.off_next_state + p] = __float_as_uint(next_state[(size_t)w * obs + p]);
    }
    if (lane == 0) {
        r[L.off_action] = (uint32_t)(int32_t)action[w];
        r[L.off_reward] = __float_as_uint(reward[w]);
        uint8_t *ids = reinterpret_cast<uint8_t *>(r + L.off_avail);
        uint32_t cnt = 0;
        for (int k = 0; k < A; k++) {
            const bool unavailable = mask ? mask[(size_t)w * A + k] != 0 : false;
            if (unavailable) continue;
            ids[cnt++] = next_avail ? (uint8_t)(int)next_avail[(size_t)w * A + k] : (uint8_t)k;
        }
        r[L.off_flags] = (terminated[w] ? 1u : 0u) | (cnt << 8);
        slots[w] = w;
    }
}

// Q(s, .) for act(): rows of plain states, every action available
__global__ void __launch_bounds__(NT, 1)
k_q_values(const float *__restrict__ net, Dims d, Plan pl, int R, int mch, int n,
           const float *__restrict__ state, float *__restrict__ out_q) {
    extern __shared__ __align__(16) float sm[];
    const int tid = threadIdx.x;
    const int r0 = blockIdx.x * R, Rv = min(R, n - r0);
    const int W = round_up(d.obs, 4);
    for (int i = tid; i < pl.total; i += NT) sm[i] = 0.f;
    __syncthreads();
    float *S = sm + pl.rec;
    for (int e = tid; e < Rv * d.obs; e += NT) {
        const int r = e / d.obs, c = e - r * d.obs;
        S[r * W + c] = state[(size_t)(r0 + r) * d.obs + c];
    }
    RowScal sc = row_scal(sm + pl.scal, R);
    if (tid < Rv) sc.cnt[tid] = d.A;
    stage_action_cols(net, d, sm + pl.WaO);
    __syncthreads();
    cta_linear<false>(S, W, Rv, net + d.oW1, d.D, d.H1, d.obs, net + d.ob1, false, sm + pl.T1t, d.H1p,
                      sm + pl.stage, sm + pl.red);
    prl_buf_layout L = {};
    all_actions_q(net, d, sm + pl.T1t, sm + pl.WaO, nullptr, 0, L, 0, Rv, mch, sc.cnt, sm + pl.Hc, sm + pl.H2c,
                  sm + pl.qa, sm + pl.stage, sm + pl.red);
    for (int e = tid; e < Rv * d.A; e += NT) out_q[(size_t)r0 * d.A + e] = sm[pl.qa + e];
}

}  // namespace

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
static const int kMaxCtas = 148;

static int64_t align_up64(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

static int check_cfg(const prl_dqn_cfg *c) {
    PRL_REQUIRE(c, "null cfg");
    PRL_REQUIRE(c->obs_dim > 0 && c->n_actions > 0 && c->n_actions <= 255, "bad obs_dim / n_actions");
    PRL_REQUIRE(c->hidden1 > 0 && c->hidden2 > 0, "two positive hidden sizes are required");
    PRL_REQUIRE(c->target_update_freq > 0, "target_update_freq must be positive");
    PRL_REQUIRE(c->max_batch > 0 && c->max_rounds > 0, "max_batch / max_rounds must be positive");
    return PRL_OK;
}

static prl_buf_layout tmp_layout(const prl_dqn_cfg *c) {
    prl_buf_desc dd;
    dd.capacity = c->max_batch;
    dd.obs_dim = c->obs_dim;
    dd.act_dim = 1;
    dd.n_actions = c->n_actions;
    dd.flags = PRL_BUF_DISCRETE | PRL_BUF_DYNAMIC_ACTIONS;
    prl_buf_layout l;
    prl_buf_layout_of(&dd, &l);
    return l;
}

extern "C" int64_t prl_dqn_param_count(const prl_dqn_cfg *c) {
    if (check_cfg(c)) return -1;
    return make_dims(c->obs_dim, c->n_actions, c->hidden1, c->hidden2).P;
}

struct WsPlan { int64_t gpart, slots, logical, scal, tmp_rec, tmp_slots, multi, is_w, td, tc_tiles, total; };
static WsPlan ws_plan(const prl_dqn_cfg *c) {
    Dims d = make_dims(c->obs_dim, c->n_actions, c->hidden1, c->hidden2);
    WsPlan w;
    int64_t o = 0;
    w.gpart = o; o = align_up64(o + (int64_t)kMaxCtas * d.Pp * 4, 256);
    w.slots = o; o = align_up64(o + (int64_t)c->max_rounds * c->max_batch * 4, 256);
    w.logical = o; o = align_up64(o + (int64_t)c->max_rounds * c->max_batch * 4, 256);
    w.scal = o; o = align_up64(o + (int64_t)c->max_rounds * 8, 256);
    w.tmp_rec = o; o = align_up64(o + tmp_layout(c).storage_bytes, 256);
    w.tmp_slots = o; o = align_up64(o + (int64_t)c->max_batch * 4, 256);
    w.multi = o; o = align_up64(o + 64 * 1024, 256);
    w.is_w = o; o = align_up64(o + (int64_t)c->max_rounds * c->max_batch * 4, 256);
    w.td = o; o = align_up64(o + (int64_t)c->max_batch * 4, 256);
    w.tc_tiles = o; o = align_up64(o + prl_tc_tile_floats(c) * 4, 256);
    w.total = o;
    return w;
}

extern "C" int64_t prl_dqn_workspace_bytes(const prl_dqn_cfg *c) {
    if (check_cfg(c)) return -1;
    return ws_plan(c).total;
}

extern "C" int prl_dqn_create(prl_dqn **out, const prl_dqn_cfg *cfg, float *w, float *w_target, float *exp_avg,
                              float *exp_avg_sq, float *max_exp_avg_sq, int64_t adam_step, void *workspace) {
    PRL_REQUIRE(out && w && w_target && exp_avg && exp_avg_sq && max_exp_avg_sq && workspace, "null argument");
    int rc = check_cfg(cfg);
    if (rc) return rc;
    PRL_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
    prl_dqn *q = new (std::nothrow) prl_dqn();
    if (!q) return fail(PRL_ENOMEM, "out of host memory");
    q->cfg = *cfg;
    q->d = make_dims(cfg->obs_dim, cfg->n_actions, cfg->hidden1, cfg->hidden2);
    q->w = w; q->wt = w_target; q->m = exp_avg; q->v = exp_avg_sq; q->vmax = max_exp_avg_sq;
    q->adam_step = adam_step;
    WsPlan ws = ws_plan(cfg);
    char *base = (char *)workspace;
    q->gpart = (float *)(base + ws.gpart);
    q->slots = (int32_t *)(base + ws.slots);
    q->logical = (int32_t *)(base + ws.logical);
    q->scal_dev = (float2 *)(base + ws.scal);
    q->tmp_rec = (uint32_t *)(base + ws.tmp_rec);
    q->tmp_slots = (int32_t *)(base + ws.tmp_slots);
    q->multi_dev = (void *)(base + ws.multi);
    q->is_w = (float *)(base + ws.is_w);
    q->td = (float *)(base + ws.td);
    q->tc_tiles = prl_tc_tile_floats(cfg) ? (float *)(base + ws.tc_tiles) : nullptr;
    q->tmp_lay = tmp_layout(cfg);
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&q->sm_count, cudaDevAttrMultiProcessorCount, dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&q->max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    // the opt-in limit covers static + dynamic shared memory: k_dqn_learn's sampler CTA keeps its MT19937 state in
    // static shared memory, so a plan has to fit in what is left (or cudaFuncSetAttribute refuses the launch)
    cudaFuncAttributes fa;
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_dqn_learn);
    if (e == cudaSuccess) q->learn_smem = q->max_smem - (int)fa.sharedSizeBytes;
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k_q_values);
    if (e == cudaSuccess) q->qv_smem = q->max_smem - (int)fa.sharedSizeBytes;
    if (e == cudaSuccess) e = q->stage.open((size_t)cfg->max_rounds * 8);
    if (e != cudaSuccess) {
        delete q;
        return fail(PRL_ECUDA, "prl_dqn_create: %s", cudaGetErrorString(e));
    }
    q->last_launches = q->last_ctas = q->last_rows = 0;
    q->timing = 0;
    q->prof = nullptr;
    q->comm = nullptr;
    q->t0 = q->t1 = nullptr;
    *out = q;
    return PRL_OK;
}

extern "C" int prl_dqn_destroy(prl_dqn *q) {
    if (!q) return PRL_OK;
    q->stage.close();
    if (q->t0) { cudaEventDestroy(q->t0); cudaEventDestroy(q->t1); }
    delete q;
    return PRL_OK;
}

extern "C" int prl_dqn_set_comm(prl_dqn *q, prl_comm *comm) {
    PRL_REQUIRE(q, "null handle");
    q->comm = comm;
    return PRL_OK;
}

extern "C" int prl_comm_create(prl_comm **out, int rank, int world, int64_t max_param_count) {
    PRL_REQUIRE(out && world >= 1 && world <= 16 && rank >= 0 && rank < world, "bad rank/world");
    PRL_REQUIRE(max_param_count > 0, "bad parameter count");
    prl_comm *c = new (std::nothrow) prl_comm();
    if (!c) return fail(PRL_ENOMEM, "out of host memory");
    c->rank = rank; c->world = world;
    c->slot_floats = (max_param_count + 63) / 64 * 64;
    c->exchanges = 0;
    c->opened = world == 1;
    for (int p = 0; p < 16; p++) { c->peer_inbox[p] = nullptr; c->peer_flags[p] = nullptr; }
    const size_t inbox_bytes = (size_t)2 * world * c->slot_floats * 8;  // (value, sequence) pairs
    cudaError_t e = cudaMalloc((void **)&c->inbox, inbox_bytes);
    if (e == cudaSuccess) e = cudaMalloc((void **)&c->flags, kCommFlags * 4);
    if (e == cudaSuccess) e = cudaMemset(c->inbox, 0, inbox_bytes);
    if (e == cudaSuccess) e = cudaMemset(c->flags, 0, kCommFlags * 4);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { delete c; return fail(PRL_ECUDA, "prl_comm_create: %s", cudaGetErrorString(e)); }
    c->peer_inbox[rank] = c->inbox;
    c->peer_flags[rank] = c->flags;
    *out = c;
    return PRL_OK;
}

extern "C" int prl_comm_local_handles(prl_comm *c, uint8_t *blob) {
    PRL_REQUIRE(c && blob, "null argument");
    static_assert(2 * sizeof(cudaIpcMemHandle_t) <= PRL_COMM_HANDLE_BYTES, "blob too small");
    cudaIpcMemHandle_t h[2];
    PRL_CUDA(cudaIpcGetMemHandle(&h[0], c->inbox));
    PRL_CUDA(cudaIpcGetMemHandle(&h[1], c->flags));
    memset(blob, 0, PRL_COMM_HANDLE_BYTES);
    memcpy(blob, h, sizeof(h));
    return PRL_OK;
}

extern "C" int prl_comm_open_peers(prl_comm *c, const uint8_t *blobs) {
    PRL_REQUIRE(c && blobs, "null argument");
    for (int p = 0; p < c->world; p++) {
        if (p == c->rank) continue;
        cudaIpcMemHandle_t h[2];
        memcpy(h, blobs + (size_t)p * PRL_COMM_HANDLE_BYTES, sizeof(h));
        PRL_CUDA(cudaIpcOpenMemHandle((void **)&c->peer_inbox[p], h[0], cudaIpcMemLazyEnablePeerAccess));
        PRL_CUDA(cudaIpcOpenMemHandle((void **)&c->peer_flags[p], h[1], cudaIpcMemLazyEnablePeerAccess));
    }
    c->opened = true;
    return PRL_OK;
}

extern "C" int prl_comm_destroy(prl_comm *c) {
    if (!c) return PRL_OK;
    for (int p = 0; p < c->world; p++) {
        if (p == c->rank) continue;
        if (c->peer_inbox[p]) cudaIpcCloseMemHandle(c->peer_inbox[p]);
        if (c->peer_flags[p]) cudaIpcCloseMemHandle(c->peer_flags[p]);
    }
    cudaFree(c->inbox);
    cudaFree(c->flags);
    delete c;
    return PRL_OK;
}

extern "C" int prl_dqn_set_timing(prl_dqn *q, int enable) {
    PRL_REQUIRE(q, "null handle");
    if (enable && !q->t0) {
        PRL_CUDA(cudaEventCreate(&q->t0));
        PRL_CUDA(cudaEventCreate(&q->t1));
    }
    q->timing = enable != 0;
    return PRL_OK;
}
extern "C" int prl_dqn_set_profile(prl_dqn *q, long long *stamps_dev) {
    PRL_REQUIRE(q, "null handle");
    q->prof = stamps_dev;
    return PRL_OK;
}
extern "C" int prl_dqn_last_kernel_ms(prl_dqn *q, float *ms) {
    PRL_REQUIRE(q && ms && q->t0, "timing was not enabled");
    PRL_CUDA(cudaEventSynchronize(q->t1));
    PRL_CUDA(cudaEventElapsedTime(ms, q->t0, q->t1));
    return PRL_OK;
}

extern "C" int64_t prl_dqn_adam_step(const prl_dqn *q) { return q ? q->adam_step : -1; }
extern "C" int prl_dqn_set_adam_step(prl_dqn *q, int64_t s) {
    PRL_REQUIRE(q && s >= 0, "bad argument");
    q->adam_step = s;
    return PRL_OK;
}
extern "C" int prl_dqn_set_lr(prl_dqn *q, double lr) {
    PRL_REQUIRE(q && lr >= 0, "bad argument");
    q->cfg.lr = lr;
    return PRL_OK;
}
extern "C" int prl_dqn_last_launch_info(const prl_dqn *q, int32_t *launches, int32_t *ctas, int32_t *rows) {
    PRL_REQUIRE(q, "null handle");
    if (launches) *launches = q->last_launches;
    if (ctas) *ctas = q->last_ctas;
    if (rows) *rows = q->last_rows;
    return PRL_OK;
}

// choose rows per CTA, target chunk rows and check shared memory
static int choose_tiling(const prl_dqn *q, int B, int W, int *R_out, int *mch_out, Plan *plan_out) {
    const Dims &d = q->d;
    int R = q->cfg.rows_per_cta;
    const int max_ctas = (q->sm_count < kMaxCtas ? q->sm_count : kMaxCtas) - 1;  // one SM for the index producer
    if (R <= 0) {
        R = 4;  // 64 target rows per CTA at A = 16: one full register-tiled block
        while ((B + R - 1) / R > max_ctas) R *= 2;
    }
    PRL_REQUIRE((B + R - 1) / R <= max_ctas, "rows_per_cta=%d needs more than %d CTAs for batch %d", R, max_ctas, B);
    PRL_REQUIRE(R <= NT, "rows_per_cta too large");
    int mch = 64;
    while (mch > 4 && mch / 2 >= R * d.A) mch /= 2;  // no point exceeding the rows that exist
    Plan pl;
    for (;; mch /= 2) {
        pl = make_plan(d, R, W, mch);
        if ((int64_t)pl.total * 4 <= q->learn_smem) break;
        if (mch <= 4)
            return fail(PRL_EUNSUPPORTED, "network/batch tile does not fit shared memory (%lld B needed, %d B available)",
                        (long long)pl.total * 4, q->learn_smem);
    }
    *R_out = R; *mch_out = mch; *plan_out = pl;
    return PRL_OK;
}

// per-round optimizer scalars exactly as torch evaluates them (Python floats -> fp32)
int prl_dqn_stage_scalars(prl_dqn *q, int rounds, cudaStream_t stream) {
    const prl_dqn_cfg &c = q->cfg;
    float2 *hs;
    int rc = q->stage.wait(&hs);
    if (rc) return rc;
    for (int r = 0; r < rounds; r++) hs[r] = adam_scal(c.lr, c.beta1, c.beta2, q->adam_step + r + 1);
    return q->stage.send(q->scal_dev, (size_t)rounds * 8, stream);
}

static int launch_learn(prl_dqn *q, const uint32_t *records, const prl_buf_layout &lay, int buf_flags,
                        const int32_t *slots, int rounds, int B, int64_t steps0, int first_update, float *out_mae,
                        float *out_q, float *out_y, cudaStream_t stream, prl_buf *sample_from = nullptr,
                        int32_t *out_logical = nullptr, const float *is_weight = nullptr, float *out_td = nullptr,
                        int prestaged_scal_offset = -1) {
    int R, mch;
    Plan pl;
    int rc = choose_tiling(q, B, lay.record_words, &R, &mch, &pl);
    if (rc) return rc;
    const prl_dqn_cfg &c = q->cfg;
    if (prestaged_scal_offset < 0) {
        rc = prl_dqn_stage_scalars(q, rounds, stream);
        if (rc) return rc;
    }

    LearnArgs a;
    a.records = records; a.lay = lay; a.buf_flags = buf_flags; a.slots = slots;
    a.w = q->w; a.wt = q->wt; a.m = q->m; a.v = q->v; a.vmax = q->vmax;
    a.gpart = q->gpart; a.scal = q->scal_dev + (prestaged_scal_offset < 0 ? 0 : prestaged_scal_offset);
    a.is_weight = is_weight; a.out_td = out_td;
    a.out_mae = out_mae; a.out_q = out_q; a.out_y = out_y;
    a.d = q->d; a.plan = pl;
    a.B = B; a.R = R; a.rounds = rounds; a.mch = mch; a.double_dqn = c.double_dqn; a.freq = c.target_update_freq;
    a.steps0 = steps0;
    a.first_update = first_update;
    a.decay = (float)(1.0 - c.lr * c.weight_decay);
    a.omb1 = (float)(1.0 - c.beta1);
    a.beta2 = (float)c.beta2;
    a.omb2 = (float)(1.0 - c.beta2);
    a.eps = (float)c.eps;
    a.gamma = (float)c.gamma;
    a.tau = (float)c.tau;
    a.omtau = (float)(1.0 - c.tau);
    a.inv_b2 = 2.0f / (float)B;
    const int G = (B + R - 1) / R;
    size_t smem = (size_t)pl.total * 4;
    a.G = G;
    a.fused_sampler = 0;
    a.mt_state = nullptr;
    a.prof = q->prof;
    a.rank = 0; a.world = 1; a.inbox = nullptr; a.flags = nullptr; a.comm_slot = 0; a.exch0 = 0; a.inv_world = 1.f;
    a.shard_world = 1; a.shard_rank = 0; a.g_oldest = 0; a.local_cap = 0;
    for (int p = 0; p < 16; p++) { a.peer_inbox[p] = nullptr; a.peer_flags[p] = nullptr; }
    if (q->comm && sample_from) {  // data-parallel learn(): exchange inside the kernel
        prl_comm *c = q->comm;
        PRL_REQUIRE(c->opened, "communicator peers were not opened");
        PRL_REQUIRE(c->slot_floats >= q->d.P, "communicator slots are smaller than the parameter vector");
        PRL_REQUIRE(G <= kCommFlags, "too many learner CTAs for the communicator");
        a.rank = c->rank; a.world = c->world; a.inbox = c->inbox; a.flags = c->flags;
        a.comm_slot = c->slot_floats; a.exch0 = c->exchanges; a.inv_world = 1.0f / (float)c->world;
        for (int p = 0; p < c->world; p++) { a.peer_inbox[p] = c->peer_inbox[p]; a.peer_flags[p] = c->peer_flags[p]; }
        c->exchanges += (unsigned long long)rounds;
        if (sample_from->shard_world > 1) {
            // replay sharded over the ranks: same B indices everywhere, each rank contributes the UNNORMALISED partial
            // gradient of the rows it owns (every row already carries 2 / B), the exchange sums them
            PRL_REQUIRE(sample_from->shard_world == c->world && sample_from->shard_rank == c->rank,
                        "replay shard (%d of %d) does not match the communicator (%d of %d)", sample_from->shard_rank,
                        sample_from->shard_world, c->rank, c->world);
            PRL_REQUIRE(c->slot_floats >= q->d.P + 1, "communicator slots must hold the parameter vector + 1");
            PRL_REQUIRE(!is_weight, "prioritized replay is not sharded here");
            a.shard_world = c->world; a.shard_rank = c->rank;
            a.g_oldest = sample_from->g_pushed - prl_buf_global_len(sample_from);
            a.local_cap = sample_from->desc.capacity;
            a.inv_world = 1.f;
        }
    } else if (sample_from && sample_from->shard_world > 1) {
        return fail(PRL_EINVAL, "a sharded replay buffer needs a learner with a communicator (set_communicator)");
    }
    if (sample_from) {  // the index stream is produced inside the kernel by CTA number G
        size_t sbytes = 0;
        rc = prl_sampler_params(sample_from, B, &a.sp, &sbytes);
        if (rc) return rc;
        a.sp.out_slot = const_cast<int32_t *>(slots);
        a.sp.out_logical = out_logical;
        a.mt_state = sample_from->mt_state;
        a.fused_sampler = 1;
        if (sbytes > smem) smem = sbytes;
        PRL_REQUIRE(smem <= (size_t)q->learn_smem, "sampler tables do not fit shared memory");
    }
    PRL_CUDA(cudaFuncSetAttribute(k_dqn_learn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    void *args[] = {(void *)&a};
    if (q->timing) PRL_CUDA(cudaEventRecord(q->t0, stream));
    PRL_CUDA(cudaLaunchCooperativeKernel((void *)k_dqn_learn, dim3(G + a.fused_sampler), dim3(NT), args, smem, stream));
    if (q->timing) PRL_CUDA(cudaEventRecord(q->t1, stream));
    q->adam_step += rounds;
    q->last_ctas = G;
    q->last_rows = R;
    return PRL_OK;
}

extern "C" int prl_dqn_learn(prl_dqn *q, prl_buf *buf, int rounds, int batch, int64_t training_steps0,
                             float *out_mae, float *out_q, float *out_y, int32_t *out_logical, void *stream_) {
    PRL_REQUIRE(q && buf && out_mae, "null argument");
    PRL_REQUIRE(rounds > 0 && rounds <= q->cfg.max_rounds, "rounds %d outside [1, max_rounds=%d]", rounds,
                q->cfg.max_rounds);
    PRL_REQUIRE(batch > 0 && batch <= q->cfg.max_batch, "batch %d outside [1, max_batch=%d]", batch,
                q->cfg.max_batch);
    PRL_REQUIRE(buf->desc.flags & PRL_BUF_DISCRETE, "DQN needs a discrete-action buffer");
    PRL_REQUIRE(buf->desc.obs_dim == q->cfg.obs_dim && buf->desc.n_actions == q->cfg.n_actions,
                "buffer (obs %d, actions %d) does not match learner (obs %d, actions %d)", buf->desc.obs_dim,
                buf->desc.n_actions, q->cfg.obs_dim, q->cfg.n_actions);
    cudaStream_t stream = (cudaStream_t)stream_;
    int rc = launch_learn(q, buf->records, buf->lay, buf->desc.flags, q->slots, rounds, batch, training_steps0,
                          (training_steps0 + 2) % q->cfg.target_update_freq == 0, out_mae, out_q, out_y, stream,
                          buf, out_logical);
    if (rc) return rc;
    q->last_launches = 1;  // one persistent kernel: index producer CTA + learner CTAs
    return PRL_OK;
}

extern "C" int prl_dqn_learn_per(prl_dqn *q, prl_buf *buf, prl_per *per, int rounds, int batch, int64_t training_steps0,
                                 float *out_mae, float *out_q, float *out_y, int32_t *out_slots, float *out_weights,
                                 void *stream_) {
    PRL_REQUIRE(q && buf && per && out_mae, "null argument");
    PRL_REQUIRE(rounds > 0 && rounds <= q->cfg.max_rounds, "rounds %d outside [1, max_rounds=%d]", rounds, q->cfg.max_rounds);
    PRL_REQUIRE(batch > 0 && batch <= q->cfg.max_batch && batch <= 1024, "batch %d outside [1, min(max_batch, 1024)]", batch);
    PRL_REQUIRE(buf->desc.flags & PRL_BUF_DISCRETE, "DQN needs a discrete-action buffer");
    PRL_REQUIRE(buf->desc.obs_dim == q->cfg.obs_dim && buf->desc.n_actions == q->cfg.n_actions, "buffer does not match the learner");
    PRL_REQUIRE(buf->len > 0, "empty replay buffer");
    cudaStream_t stream = (cudaStream_t)stream_;
    int rc = prl_dqn_stage_scalars(q, rounds, stream);
    if (rc) return rc;
    for (int r = 0; r < rounds; r++) {
        int32_t *slots = q->slots + (size_t)r * batch;
        float *w = q->is_w + (size_t)r * batch;
        rc = prl_per_sample(per, batch, slots, w, stream_);
        if (rc) return rc;
        const int64_t s0 = training_steps0 + r;
        rc = launch_learn(q, buf->records, buf->lay, buf->desc.flags, slots, 1, batch, s0,
                          (s0 + 2) % q->cfg.target_update_freq == 0, out_mae + r, out_q ? out_q + (size_t)r * batch : nullptr,
                          out_y ? out_y + (size_t)r * batch : nullptr, stream, nullptr, nullptr, w, q->td, r);
        if (rc) return rc;
        rc = prl_per_set_priorities(per, slots, q->td, batch, nullptr, stream_);
        if (rc) return rc;
    }
    if (out_slots) PRL_CUDA(cudaMemcpyAsync(out_slots, q->slots, (size_t)rounds * batch * 4, cudaMemcpyDeviceToDevice, stream));
    if (out_weights) PRL_CUDA(cudaMemcpyAsync(out_weights, q->is_w, (size_t)rounds * batch * 4, cudaMemcpyDeviceToDevice, stream));
    q->last_launches = 3 * rounds;
    return PRL_OK;
}

extern "C" int prl_dqn_learn_batch(prl_dqn *q, int batch, const float *state, const int64_t *action,
                                   const float *reward, const float *next_state, const uint8_t *terminated,
                                   const float *next_avail, const uint8_t *next_unavail_mask, int do_target_update,
                                   float *out_mae, float *out_q, float *out_y, void *stream_) {
    PRL_REQUIRE(q && state && action && reward && next_state && terminated && out_mae, "null argument");
    PRL_REQUIRE(batch > 0 && batch <= q->cfg.max_batch, "batch %d outside [1, max_batch=%d]", batch,
                q->cfg.max_batch);
    cudaStream_t stream = (cudaStream_t)stream_;
    const int threads = 256, blocks = (batch * 32 + threads - 1) / threads;
    k_pack_batch<<<blocks, threads, 0, stream>>>(q->tmp_rec, q->tmp_lay, q->cfg.obs_dim, q->cfg.n_actions, batch,
                                                 state, (const long long *)action, reward, next_state, terminated,
                                                 next_avail, next_unavail_mask, q->tmp_slots);
    PRL_CUDA(cudaGetLastError());
    int rc = launch_learn(q, q->tmp_rec, q->tmp_lay, PRL_BUF_DISCRETE | PRL_BUF_DYNAMIC_ACTIONS, q->tmp_slots, 1,
                          batch, 0, do_target_update != 0, out_mae, out_q, out_y, stream);
    if (rc) return rc;
    q->last_launches = 2;
    return PRL_OK;
}

extern "C" int prl_dqn_q_values(prl_dqn *q, int n, const float *state, int target, float *out_q, void *stream_) {
    PRL_REQUIRE(q && state && out_q, "null argument");
    if (n <= 0) return PRL_OK;
    const Dims &d = q->d;
    const int R = 4, W = round_up(d.obs, 4);
    int mch = 64;
    while (mch > 4 && mch / 2 >= R * d.A) mch /= 2;
    Plan pl;
    for (;; mch /= 2) {
        pl = make_plan(d, R, W, mch);
        if ((int64_t)pl.total * 4 <= q->qv_smem) break;
        if (mch <= 4) return fail(PRL_EUNSUPPORTED, "network does not fit shared memory");
    }
    const size_t smem = (size_t)pl.total * 4;
    PRL_CUDA(cudaFuncSetAttribute(k_q_values, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_q_values<<<(n + R - 1) / R, NT, smem, (cudaStream_t)stream_>>>(target ? q->wt : q->w, d, pl, R, mch, n, state,
                                                                    out_q);
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}
