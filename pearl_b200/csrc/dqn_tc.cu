// dqn_tc.cu — tensor-core DQN learner: ONE SM (one CTA) runs one complete learner, every dense
// contraction of the step on Hopper's warpgroup tensor-core instruction (wgmma, 3xTF32, fp32 accumulators in
// registers), so that a launch with L CTAs trains L independent learners (seeds / agents) concurrently — the
// aggregate mode that fills the chip — and a single learner needs one SM instead of a cooperative grid.
//
// Same semantics as the cooperative SIMT kernel in dqn.cu (DeepQLearning.learn: sample -> Q(s,a) ->
// max_a' Q_target(s',a') -> MSE -> backward -> AdamW(amsgrad) -> scheduled soft target update; reference
// call sites in include/pearl_b200.h).  Supported shape class: two hidden layers of 64, obs % 8 == 0,
// obs <= 128, n_actions in {1,2,4,8,16}, batch in {128, 256}; everything else stays on the SIMT kernel.
//
// Per gradient step (256 threads = two warpgroups; warpgroup h owns the 64 batch rows 128 i + 64 h .. of row tile i,
// a thread the elements of those rows that the wgmma accumulator layout gives it, umma.cuh):
//   layer 1  T1 = X W1s^T: the rows are gathered into shared memory by cp.async (K chunks of 64) and read back
//            as register A fragments (RS form); B = the W1 tile.
//   phase T  target net: per action slot one 64 x 64 x 64 product whose A operand relu(T1 + W1a[:,a] + b1) is
//            built in registers from the layer-1 accumulator and never leaves them; running max over the slots.
//   phase O  online net forward the same way, loss gradient, dZ2, dH1 = dZ2 W2 (B operand = W2^T tile), all on
//            register operands; then the weight gradients as products over the batch dimension:
//            dW2 = dZ2^T H1, dW1s = dZ1^T S, and [db | dW1a] = dZ^T E with E = [1 | onehot(action)];
//            their operands are explicitly transposed tiles written with a 144-byte chunk pitch
//            (bank-conflict-free column scatter), 64 batch rows per pass, the two warpgroups taking
//            different output columns.  Their accumulators stay in registers for the whole step.
//   AdamW    gradients registers -> shared staging, then one coalesced 16-byte sweep over the flat parameter
//            vector (parameters / moments in L2) that also writes the operand-layout weight tiles.
//
// The weights are kept in global memory a second time IN THE OPERAND LAYOUT (hi tile = the fp32 values — the tensor
// core truncates them to TF32 — and lo tile = x - trunc_tf32(x)), written by AdamW / the soft target update next to the
// flat torch-order vectors, so staging a network's B operands is three TMA bulk copies (cp.async.bulk + mbarrier
// complete_tx) issued by one thread.  The W2 tiles store their K axis in the order umma::kperm, which is the order in
// which an accumulator's columns feed the next product's register A operand.  The target network's small vectors are
// cached in shared memory between soft updates, AdamW walks one flat list with two groups of loads in flight, the soft
// target update is applied to the tiles in tile order.
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>

#include <new>

#include "dqn_common.cuh"
#include "sampler.cuh"
#include "umma.cuh"

using namespace prl;

int prl_sampler_params(const prl_buf *b, int k, prl::SamplerParams *sp, size_t *smem_bytes);

namespace {

constexpr int NTH = 256;
constexpr int HID = 64;
constexpr int MAX_B = 256;
// shared memory regions (bytes): 1 = W1 hi | lo tiles, 2 = row staging of layer 1 / gradient staging of AdamW,
// 3 = W2 hi | lo | W2^T hi | lo tiles
constexpr int REG1 = 0, REG2 = 65536, REG3 = 131072, MISC_OFF = 196608;
constexpr int HALF = 32768;          // hi tile at region base, lo tile at base + HALF
constexpr int SBUF = 16384;          // layer-1 row staging of one warpgroup: [64 rows][64 floats]
// transposed-tile arena (regions 1+2) for the weight-gradient products, 64 batch rows per pass
constexpr int TL = 144;              // chunk pitch of transposed tiles
constexpr int AR_A_HI = 0, AR_A_LO = 18432, AR_B_HI = 36864, AR_B_LO = 73728, AR_E = 110592;

struct TcLearner {            // one per CTA, in global memory
    const uint32_t *records;
    float *tiles;             // operand-layout weight tiles: online net, then target net (net_tile_floats each)
    const int32_t *slots;     // [rounds][B]
    float *w, *wt, *m, *v, *vmax;
    const float2 *scal;       // [rounds]
    float *out_mae, *out_q, *out_y;
    long long steps0;
    int buf_flags;
    int pad_;
};

struct TcArgs {
    const TcLearner *learners;
    prl_buf_layout lay;
    Dims d;
    int B, rounds, freq;
    int round0;        // this launch runs rounds [round0, round0 + rounds) of the call (chunked launches)
    float decay, omb1, beta2, omb2, eps, gamma, tau, omtau, inv_b2;
    long long *prof;   // optional [rounds][16] SM-clock stamps of one CTA
    int prof_cta;      // which CTA writes them (PRL_TC_PROF_CTA, default 0: the learners do not all run at the same speed)
};

#define TC_STAMP(idx)                                                                          \
    do {                                                                                       \
        if (a.prof && blockIdx.x == a.prof_cta && threadIdx.x == 0) a.prof[(size_t)round * 16 + (idx)] = clock64(); \
    } while (0)

struct Misc {
    // small fp32 vectors of a network: W1[:, obs + a] + b1, b2, w3, b3.  [0] online, [1] target (the target's only change at
    // a scheduled soft update, so they are loaded then and in the prologue, not every round)
    struct Smalls { float watb[16][HID]; float b2[HID], w3[HID]; float b3, pad0[3]; } sm[2];
    float y[MAX_B];
    int act[MAX_B], cnt[MAX_B], slot[MAX_B];
    float rew[MAX_B], term[MAX_B];
    float redw[8][HID];
    float redmae[8], reddb3[8];
    unsigned long long bar[3];   // 0: target tiles; 1: online W1 tiles; 2: online W2 tiles
};

__device__ __forceinline__ void cp_async16_zfill_tc(void *smem_dst, const void *gmem_src, int src_bytes) {
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(sa), "l"(gmem_src), "r"(src_bytes) : "memory");
}

__device__ __forceinline__ void group_sync(int g) { asm volatile("bar.sync %0, %1;" ::"r"(1 + g), "r"(128) : "memory"); }

__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(umma::smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA bulk copy global -> shared, completion counted in bytes on `bar`
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(umma::smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(umma::smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
using umma::tf32_lo;

// Operand-layout copies of one network's matrices in global memory (floats):
//   [W1 hi: 64 x obs][W1 lo][W2 hi: 64 x 64][W2 lo]      (the shared-memory images, tile by tile; the W2 tiles with their
//   K axis in umma::kperm order; the W2^T tiles of the online network are transposed out of the W2 tiles in shared memory)
struct NetTiles { float *w1hi, *w1lo, *w2; };   // w2: the 2 x 4096-float block W2 hi | W2 lo
__host__ __device__ inline int net_tile_floats(int obs) { return 128 * obs + 2 * HID * HID; }
__device__ __forceinline__ NetTiles net_tiles(float *base, int obs) { return NetTiles{base, base + 64 * obs, base + 128 * obs}; }
// all tiles of one network from its flat parameter vector (kernel prologue, soft target update)
__device__ void rebuild_tiles(const float *__restrict__ net, const Dims &d, const NetTiles &t, int tid) {
    for (int e = tid; e < HID * d.obs; e += NTH) {
        const int j = e / d.obs, k = e - j * d.obs;
        const float x = __ldcg(net + d.oW1 + (size_t)j * d.D + k);
        const int idx = umma::tile_index(j, k, d.obs);
        t.w1hi[idx] = x; t.w1lo[idx] = tf32_lo(x);
    }
    for (int e = tid; e < HID * HID; e += NTH) {
        const int j = e >> 6, k = e & 63;
        const float x = __ldcg(net + d.oW2 + e);
        const int i1 = umma::tile_index(j, umma::kperm(k), HID);
        t.w2[i1] = x; t.w2[4096 + i1] = tf32_lo(x);
    }
}
// the small fp32 vectors of a network (action columns + b1, b2, w3, b3); all loads of a thread issued before the first use
__device__ void load_smalls(const float *__restrict__ net, const Dims &d, Misc::Smalls &mi) {
    const int tid = threadIdx.x;
    float wa[4], bb[4];                                           // A * 64 <= 1024 elements: <= 4 per thread
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int e = tid + u * NTH;
        if (e < d.A * HID) {
            const int j = e / d.A, a = e - j * d.A;
            wa[u] = __ldcg(net + d.oW1 + (size_t)j * d.D + d.obs + a);
            bb[u] = __ldcg(net + d.ob1 + j);
        }
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
        const int e = tid + u * NTH;
        if (e < d.A * HID) { const int j = e / d.A, a = e - j * d.A; mi.watb[a][j] = wa[u] + bb[u]; }
    }
    if (tid < HID) { mi.b2[tid] = __ldcg(net + d.ob2 + tid); mi.w3[tid] = __ldcg(net + d.oW3 + tid); }
    if (tid == 0) mi.b3 = __ldcg(net + d.ob3);
}

__device__ __forceinline__ float fast_sqrt(float x) {
    float r;
    asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
struct AdamScalarsTc : AdamScalars { float inv_bc2_sqrt; };

__device__ __forceinline__ float adam_math(float w, float &m, float &v, float &x, float g, const AdamScalarsTc &hs) {
    float p = __fmul_rn(w, hs.decay);
    m = fmaf(hs.omb1, g - m, m);
    v = __fadd_rn(__fmul_rn(v, hs.beta2), __fmul_rn(__fmul_rn(hs.omb2, g), g));
    x = fmaxf(x, v);
    // one SM updates all 13.5k parameters: MUFU sqrt / divide (<= 2 ulp) instead of the IEEE
    // software sequences; well inside the 1e-4 parity budget
    const float denom = __fadd_rn(__fmul_rn(fast_sqrt(x), hs.inv_bc2_sqrt), hs.eps);
    return __fadd_rn(p, __fdividef(__fmul_rn(-hs.step_size, m), denom));
}

// t1[64 x 64] = X[rows row0 .. row0 + 64) W1s^T for this warpgroup, X = state (online) or next_state (target).  The rows
// arrive by coalesced 16-byte cp.async (16 lanes per row) in a staging buffer [64 rows][64 floats] whose 16-byte chunk c
// of row r sits at chunk position c ^ (r & 7), which makes the fragment reads below (8 rows x 4 consecutive k per warp
// and load) conflict free; 64 columns of K per pass.
__device__ __forceinline__ void layer1_block(const TcArgs &a, const TcLearner &L, const Misc &mi, char *smem, int field_off, int row0,
                                             float (&t1)[32]) {
    const int m = threadIdx.x & 127, g = threadIdx.x >> 7, t = threadIdx.x & 3;
    const umma::Tile B_hi = umma::make_tile(smem + REG1, a.d.obs, 128), B_lo = umma::make_tile(smem + REG1 + HALF, a.d.obs, 128);
    float *sbuf = reinterpret_cast<float *>(smem + REG2 + g * SBUF);
    for (int kc = 0; kc * 64 < a.d.obs; kc++) {
#pragma unroll 4
        for (int i = 0; i < 8; i++) {
            const int item = i * 128 + m, rr = item >> 4, c = item & 15, k = kc * 64 + c * 4;
            const float *src = reinterpret_cast<const float *>(L.records + (size_t)mi.slot[row0 + rr] * a.lay.record_words) + field_off + k;
            const int nb = k < a.d.obs ? 16 : 0;
            cp_async16_zfill_tc(sbuf + rr * 64 + ((c ^ (rr & 7)) << 2), nb ? src : reinterpret_cast<const float *>(L.records), nb);
        }
        cp_async_commit();
        cp_async_wait<0>();
        group_sync(g);
        float hi[32], lo[32];
#pragma unroll
        for (int ks = 0; ks < 8; ks++)
#pragma unroll
            for (int q = 0; q < 2; q++)
#pragma unroll
                for (int p = 0; p < 2; p++) {
                    const int r = umma::acc_row(p), k = 8 * ks + t + 4 * q;
                    umma::split_tf32(sbuf[r * 64 + (((k >> 2) ^ (r & 7)) << 2) + (k & 3)], hi[4 * ks + 2 * q + p], lo[4 * ks + 2 * q + p]);
                }
        const int keff = min(64, a.d.obs - kc * 64);
        umma::gemm3_rs<HID, 8>(t1, hi, lo, B_hi.shifted(kc * 2048), B_lo.shifted(kc * 2048), kc > 0, keff >> 3);
        umma::wg_commit();
        umma::wg_wait<0>();
        group_sync(g);   // the staging buffer is free for the next pass
    }
}

// register A fragments (hi / lo) of the next product from values in accumulator order: v[4 j + 2 p + e] -> a[4 j + 2 e + p]
__device__ __forceinline__ void acc_to_frag(const float (&v)[32], float (&hi)[32], float (&lo)[32]) {
#pragma unroll
    for (int j = 0; j < 8; j++)
#pragma unroll
        for (int p = 0; p < 2; p++)
#pragma unroll
            for (int e = 0; e < 2; e++) umma::split_tf32(v[4 * j + 2 * p + e], hi[4 * j + 2 * e + p], lo[4 * j + 2 * e + p]);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// d[64 x n] (+)= A B^T over 64 batch rows, n in {8, 16, 32, 64}
__device__ __forceinline__ void gemm3_n(int n, float *d, umma::Tile ah, umma::Tile al, umma::Tile bh, umma::Tile bl, bool accumulate) {
    if (n == 64) umma::gemm3<64>(d, ah, al, bh, bl, 64, accumulate);
    else if (n == 32) umma::gemm3<32>(d, ah, al, bh, bl, 64, accumulate);
    else if (n == 16) umma::gemm3<16>(d, ah, al, bh, bl, 64, accumulate);
    else umma::gemm3<8>(d, ah, al, bh, bl, 64, accumulate);
}
__host__ __device__ inline int pow2_cols(int n) { return n > 32 ? 64 : n > 16 ? 32 : n > 8 ? 16 : 8; }

__global__ void __launch_bounds__(NTH, 1) k_dqn_tc(const TcArgs a) {
    extern __shared__ __align__(1024) char smem[];
    Misc &mi = *reinterpret_cast<Misc *>(smem + MISC_OFF);
    TcLearner L = a.learners[blockIdx.x];
    if (a.round0) {   // a later chunk of the same call: shift every per-round array once
        L.slots += (size_t)a.round0 * a.B;
        L.scal += a.round0;
        L.out_mae += a.round0;
        if (L.out_q) L.out_q += (size_t)a.round0 * a.B;
        if (L.out_y) L.out_y += (size_t)a.round0 * a.B;
        L.steps0 += a.round0;
    }
    const Dims &d = a.d;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int h = tid >> 7, t4 = tid & 3;
    const int ntiles = a.B >> 7;
    const int W = a.lay.record_words;
    const int rA = umma::acc_row(0), rB = umma::acc_row(1);   // this thread's two rows of its warpgroup's 64-row block

    // De-phase the learners: identical CTAs started together run in lock-step and hit L2 / HBM with their AdamW sweeps
    // (432 KB each) and row gathers all at once; a start offset of up to ~50 us spreads those bursts over the round.
    if (tid == 0 && gridDim.x > 1) {
        const long long t0 = clock64(), wait = (long long)(blockIdx.x % 48) * 2000;
        while (clock64() - t0 < wait) __nanosleep(100);
    }
    uint64_t *bar = reinterpret_cast<uint64_t *>(mi.bar);
    if (tid == 0)
        for (int i = 0; i < 3; i++) umma::mbar_init(bar + i, 1);
    // the operand-layout tiles follow the flat parameters (which the host may have changed between calls)
    const NetTiles To = net_tiles(L.tiles, d.obs), Tt = net_tiles(L.tiles + net_tile_floats(d.obs), d.obs);
    rebuild_tiles(L.w, d, To, tid);
    rebuild_tiles(L.wt, d, Tt, tid);
    fence_proxy_async_all();
    __syncthreads();
    const uint32_t w1_bytes = 64u * d.obs * 4, w2_bytes = 2u * HID * HID * 4;
    // B-operand tiles of one network by TMA: W1 hi / lo into region 1, the W2 block into region 3
    auto tma_w1 = [&](const NetTiles &t, uint64_t *b) {
        mbar_expect_tx(b, 2 * w1_bytes);
        bulk_g2s(smem + REG1, t.w1hi, w1_bytes, b);
        bulk_g2s(smem + REG1 + HALF, t.w1lo, w1_bytes, b);
    };
    auto tma_w2 = [&](const NetTiles &t, uint64_t *b) {
        mbar_expect_tx(b, w2_bytes);
        bulk_g2s(smem + REG3, t.w2, w2_bytes, b);
    };
    uint32_t par_w1 = 0;   // phase parity of bar[1] (one completion per row tile)
    const umma::Tile W2_hi = umma::make_tile(smem + REG3, 64, 128), W2_lo = umma::make_tile(smem + REG3 + 16384, 64, 128);
    const umma::Tile W2T_hi = umma::make_tile(smem + REG3 + 32768, 64, 128), W2T_lo = umma::make_tile(smem + REG3 + 49152, 64, 128);
    // weight-gradient products: warpgroup 0 accumulates dW2 (g1) and columns [0, 64) of dW1s (g2), warpgroup 1
    // [db2 | .] (g1[0..16)), [db1 | dW1a] (g1[16..32)) and columns [64, obs) of dW1s (g2)
    const int n_dw1 = h == 0 ? pow2_cols(min(d.obs, 64)) : (d.obs > 64 ? pow2_cols(d.obs - 64) : 0);

    for (int round = 0; round < a.rounds; round++) {
        TC_STAMP(0);
        // ---- per-round row scalars + L2 prefetch of the NEXT round's transitions
        if (tid < a.B) {
            const int slot = L.slots[(size_t)round * a.B + tid];
            const uint32_t *r = L.records + (size_t)slot * W;
            mi.slot[tid] = slot;
            mi.act[tid] = (int)r[a.lay.off_action];
            mi.rew[tid] = __uint_as_float(r[a.lay.off_reward]);
            const uint32_t fl = r[a.lay.off_flags];
            mi.term[tid] = (fl & 1u) ? 1.f : 0.f;
            mi.cnt[tid] = (int)((fl >> 8) & 0xffffu);
            if (round + 1 < a.rounds) {
                const char *nx = reinterpret_cast<const char *>(L.records + (size_t)L.slots[(size_t)(round + 1) * a.B + tid] * W);
                for (int o = 0; o < W * 4; o += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(nx + o));
            }
        }
        // ---- scheduled soft target update happens BEFORE this round's gradient step
        //      (deep_td_learning.py:283-284: (training_steps + 1) % freq == 0)
        const bool soft_upd = (L.steps0 + round + 2) % a.freq == 0;
        if (soft_upd) {
            for (int i = tid; i < d.P; i += NTH) L.wt[i] = soft_update(__ldcg(L.w + i), __ldcg(L.wt + i), a.tau, a.omtau);
            // The operand-layout tiles get the same elementwise update IN TILE ORDER (the hi tiles hold exactly the fp32 values of
            // the flat vectors, permuted; lo = residual of the new value): coalesced 16-byte accesses instead of rebuilding the
            // target tiles from the flat vector with scattered 4-byte stores.  Same function of the same inputs: bit-identical.
            auto update_tile = [&](const float *on_hi, float *tg_hi, float *tg_lo, int n) {
                for (int i = tid * 4; i < n; i += NTH * 4) {
                    const float4 w = __ldcg(reinterpret_cast<const float4 *>(on_hi + i)), t = __ldcg(reinterpret_cast<const float4 *>(tg_hi + i));
                    const float4 r = make_float4(soft_update(w.x, t.x, a.tau, a.omtau), soft_update(w.y, t.y, a.tau, a.omtau),
                                                 soft_update(w.z, t.z, a.tau, a.omtau), soft_update(w.w, t.w, a.tau, a.omtau));
                    *reinterpret_cast<float4 *>(tg_hi + i) = r;
                    *reinterpret_cast<float4 *>(tg_lo + i) = make_float4(tf32_lo(r.x), tf32_lo(r.y), tf32_lo(r.z), tf32_lo(r.w));
                }
            };
            update_tile(To.w1hi, Tt.w1hi, Tt.w1lo, HID * d.obs);
            update_tile(To.w2, Tt.w2, Tt.w2 + HID * HID, HID * HID);
            fence_proxy_async_all();
        }
        __syncthreads();

        // ================= phase T: y = max_a' Q_target(s', a') * gamma * (1 - term) + r =================
        TC_STAMP(1);
        if (tid == 0) {   // target tiles: three TMA bulk copies (regions 1 and 3 are free: every product of the last round was waited for)
            mbar_expect_tx(bar + 0, 2 * w1_bytes + w2_bytes);
            bulk_g2s(smem + REG1, Tt.w1hi, w1_bytes, bar + 0);
            bulk_g2s(smem + REG1 + HALF, Tt.w1lo, w1_bytes, bar + 0);
            bulk_g2s(smem + REG3, Tt.w2, w2_bytes, bar + 0);
        }
        if (soft_upd || round == 0) load_smalls(L.wt, d, mi.sm[1]);   // the target's small vectors only change at a soft update
        umma::mbar_wait(bar + 0, round & 1);
        __syncthreads();
        TC_STAMP(2);
        for (int i = 0; i < ntiles; i++) {
            const int row0 = i * 128 + h * 64;
            float t1[32];
            layer1_block(a, L, mi, smem, a.lay.off_next_state, row0, t1);
            const int rows[2] = {row0 + rA, row0 + rB};
            int cnt[2];
            const uint8_t *ids[2];
            float best[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int p = 0; p < 2; p++) {
                cnt[p] = mi.cnt[rows[p]];
                ids[p] = reinterpret_cast<const uint8_t *>(L.records + (size_t)mi.slot[rows[p]] * W + a.lay.off_avail);
            }
            for (int act = 0; act < d.A; act++) {
                float hi[32], lo[32], acc[32];
#pragma unroll
                for (int p = 0; p < 2; p++) {
                    int id = act;
                    if ((L.buf_flags & PRL_BUF_DYNAMIC_ACTIONS) && act < cnt[p]) id = ids[p][act];
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const float2 wv = *reinterpret_cast<const float2 *>(&mi.sm[1].watb[id][8 * j + 2 * t4]);
                        umma::split_tf32(fmaxf(t1[4 * j + 2 * p] + wv.x, 0.f), hi[4 * j + p], lo[4 * j + p]);
                        umma::split_tf32(fmaxf(t1[4 * j + 2 * p + 1] + wv.y, 0.f), hi[4 * j + 2 + p], lo[4 * j + 2 + p]);
                    }
                }
                umma::gemm3_rs<HID, 8>(acc, hi, lo, W2_hi, W2_lo, false);
                umma::wg_commit();
                umma::wg_wait<0>();
                float q[2] = {0.f, 0.f};
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const float2 w3v = *reinterpret_cast<const float2 *>(&mi.sm[1].w3[8 * j + 2 * t4]);
                    const float2 b2v = *reinterpret_cast<const float2 *>(&mi.sm[1].b2[8 * j + 2 * t4]);
#pragma unroll
                    for (int p = 0; p < 2; p++) {
                        q[p] = fmaf(w3v.x, fmaxf(acc[4 * j + 2 * p] + b2v.x, 0.f), q[p]);
                        q[p] = fmaf(w3v.y, fmaxf(acc[4 * j + 2 * p + 1] + b2v.y, 0.f), q[p]);
                    }
                }
#pragma unroll
                for (int p = 0; p < 2; p++) {
                    float v = quad_sum(q[p]) + mi.sm[1].b3;
                    if (act >= cnt[p]) v = -INFINITY;   // next_state_action_values[mask] = -inf
                    best[p] = fmaxf(best[p], v);
                }
            }
            if (t4 == 0)
#pragma unroll
                for (int p = 0; p < 2; p++)
                    mi.y[rows[p]] = __fadd_rn(__fmul_rn(__fmul_rn(best[p], a.gamma), 1.f - mi.term[rows[p]]), mi.rew[rows[p]]);
        }
        __syncthreads();   // both warpgroups are done with the target tiles

        // ================= phase O: online forward, loss, backward =================
        TC_STAMP(3);
        if (tid == 0) { tma_w1(To, bar + 1); tma_w2(To, bar + 2); }
        load_smalls(L.w, d, mi.sm[0]);
        umma::mbar_wait(bar + 2, round & 1);
        {   // W2^T tiles (B operand of dH1 = dZ2 W2, contraction over W2's rows) out of the W2 tiles
            const float *w2 = reinterpret_cast<const float *>(smem + REG3);
            float *w2t = reinterpret_cast<float *>(smem + REG3 + 32768);
            for (int e = tid; e < HID * HID; e += NTH) {
                const int j = e >> 6, k = e & 63, i1 = umma::tile_index(j, umma::kperm(k), HID), i2 = umma::tile_index(k, umma::kperm(j), HID);
                w2t[i2] = w2[i1]; w2t[4096 + i2] = w2[4096 + i1];
            }
            umma::fence_async_smem();
        }
        TC_STAMP(4);
        float dw3[16], g1[32], g2[32];
        float mae_acc = 0.f, db3_acc = 0.f;
#pragma unroll
        for (int c = 0; c < 16; c++) dw3[c] = 0.f;
        float *arena = reinterpret_cast<float *>(smem);
        const umma::Tile TA_hi = umma::make_tile(smem + AR_A_HI, 64, TL), TA_lo = umma::make_tile(smem + AR_A_LO, 64, TL);
        const umma::Tile TB_hi = umma::make_tile(smem + AR_B_HI, 64, TL), TB_lo = umma::make_tile(smem + AR_B_LO, 64, TL);
        const umma::Tile TE = umma::make_tile(smem + AR_E, 64, TL);
        for (int i = 0; i < ntiles; i++) {
            if (i > 0 && tid == 0) tma_w1(To, bar + 1);   // the arena of the last tile overwrote region 1
            umma::mbar_wait(bar + 1, par_w1);
            par_w1 ^= 1;
            __syncthreads();   // also: the W2^T tiles are complete
            const int row0 = i * 128 + h * 64;
            const int rows[2] = {row0 + rA, row0 + rB};
            float h1[32], z[32], hi[32], lo[32];
            layer1_block(a, L, mi, smem, a.lay.off_state, row0, h1);
            if (i == 0) TC_STAMP(5);
            int ai[2];
#pragma unroll
            for (int p = 0; p < 2; p++) {
                ai[p] = mi.act[rows[p]];
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const float2 wv = *reinterpret_cast<const float2 *>(&mi.sm[0].watb[ai[p]][8 * j + 2 * t4]);
                    h1[4 * j + 2 * p] = fmaxf(h1[4 * j + 2 * p] + wv.x, 0.f);
                    h1[4 * j + 2 * p + 1] = fmaxf(h1[4 * j + 2 * p + 1] + wv.y, 0.f);
                }
            }
            acc_to_frag(h1, hi, lo);
            umma::gemm3_rs<HID, 8>(z, hi, lo, W2_hi, W2_lo, false);
            umma::wg_commit();
            umma::wg_wait<0>();
            float part[2] = {0.f, 0.f}, dq[2];
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const float2 w3v = *reinterpret_cast<const float2 *>(&mi.sm[0].w3[8 * j + 2 * t4]);
                const float2 b2v = *reinterpret_cast<const float2 *>(&mi.sm[0].b2[8 * j + 2 * t4]);
#pragma unroll
                for (int p = 0; p < 2; p++) {
                    z[4 * j + 2 * p] = fmaxf(z[4 * j + 2 * p] + b2v.x, 0.f);
                    z[4 * j + 2 * p + 1] = fmaxf(z[4 * j + 2 * p + 1] + b2v.y, 0.f);
                    part[p] = fmaf(w3v.x, z[4 * j + 2 * p], part[p]);
                    part[p] = fmaf(w3v.y, z[4 * j + 2 * p + 1], part[p]);
                }
            }
#pragma unroll
            for (int p = 0; p < 2; p++) {
                const float q = quad_sum(part[p]) + mi.sm[0].b3;
                const float y = mi.y[rows[p]];
                dq[p] = (q - y) * a.inv_b2;
                if (t4 == 0) {
                    if (L.out_q) L.out_q[(size_t)round * a.B + rows[p]] = q;
                    if (L.out_y) L.out_y[(size_t)round * a.B + rows[p]] = y;
                    mae_acc += fabsf(q - y);
                    db3_acc += dq[p];
                }
            }
            // dW3 partial sums over this thread's two rows, then dZ2 in place of h2
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const float2 w3v = *reinterpret_cast<const float2 *>(&mi.sm[0].w3[8 * j + 2 * t4]);
                dw3[2 * j] += dq[0] * z[4 * j] + dq[1] * z[4 * j + 2];
                dw3[2 * j + 1] += dq[0] * z[4 * j + 1] + dq[1] * z[4 * j + 3];
#pragma unroll
                for (int p = 0; p < 2; p++) {
                    z[4 * j + 2 * p] = z[4 * j + 2 * p] > 0.f ? dq[p] * w3v.x : 0.f;
                    z[4 * j + 2 * p + 1] = z[4 * j + 2 * p + 1] > 0.f ? dq[p] * w3v.y : 0.f;
                }
            }
            float dz1[32];
            acc_to_frag(z, hi, lo);
            umma::gemm3_rs<HID, 8>(dz1, hi, lo, W2T_hi, W2T_lo, false);   // dH1 = dZ2 W2
            umma::wg_commit();
            umma::wg_wait<0>();
#pragma unroll
            for (int c = 0; c < 32; c++) dz1[c] = (h1[c] > 0.f) ? dz1[c] : 0.f;
            if (i == 0) TC_STAMP(6);

            // ---- weight gradients: contractions over the batch rows, 64 rows (one warpgroup's block) per pass
            for (int hf = 0; hf < 2; hf++) {
                const bool mine = h == hf;
                const bool first = (i == 0 && hf == 0);
                __syncthreads();   // previous products have been waited for: the arena is free
                if (mine) {
#pragma unroll
                    for (int j = 0; j < 8; j++)
#pragma unroll
                        for (int p = 0; p < 2; p++)
#pragma unroll
                            for (int e = 0; e < 2; e++) {
                                const int idx = umma::tile_index2(8 * j + 2 * t4 + e, p ? rB : rA, 64, TL), c = 4 * j + 2 * p + e;
                                arena[AR_A_HI / 4 + idx] = z[c]; arena[AR_A_LO / 4 + idx] = tf32_lo(z[c]);       // dZ2^T
                                arena[AR_B_HI / 4 + idx] = h1[c]; arena[AR_B_LO / 4 + idx] = tf32_lo(h1[c]);     // H1^T
                            }
#pragma unroll
                    for (int p = 0; p < 2; p++)
#pragma unroll
                        for (int x = 0; x < 8; x++) {                 // E^T: [1 | onehot(action)]
                            const int er = t4 * 8 + x;
                            arena[AR_E / 4 + umma::tile_index2(er, p ? rB : rA, 64, TL)] = (er == 0 || er == ai[p] + 1) ? 1.f : 0.f;
                        }
                }
                umma::fence_async_smem();
                __syncthreads();
                if (h == 0) umma::gemm3<64>(g1, TA_hi, TA_lo, TB_hi, TB_lo, 64, !first);
                else umma::gemm3<32>(g1, TA_hi, TA_lo, TE, TE, 64, !first, false, true);
                umma::wg_commit();
                // S^T: every warp reads whole state rows of this half coalesced (lane = k) and scatters them into column rq of
                // the transposed tile; the first four rows are requested BEFORE waiting for the dW2 product
                float sv[4][4];
                auto st_rows_load = [&](int r0) {
#pragma unroll
                    for (int ri = 0; ri < 4; ri++) {
                        const int rq = warp + 8 * (r0 + ri);
                        const float *src = reinterpret_cast<const float *>(L.records + (size_t)mi.slot[i * 128 + hf * 64 + rq] * W) + a.lay.off_state;
#pragma unroll
                        for (int jj = 0; jj < 4; jj++) sv[ri][jj] = (lane + 32 * jj < d.obs) ? __ldg(src + lane + 32 * jj) : 0.f;
                    }
                };
                auto st_rows_scatter = [&](int r0) {
#pragma unroll
                    for (int ri = 0; ri < 4; ri++) {
                        const int rq = warp + 8 * (r0 + ri);
#pragma unroll
                        for (int jj = 0; jj < 4; jj++)
                            if (lane + 32 * jj < d.obs) {
                                const int idx = umma::tile_index2(lane + 32 * jj, rq, 64, TL);
                                arena[AR_B_HI / 4 + idx] = sv[ri][jj]; arena[AR_B_LO / 4 + idx] = tf32_lo(sv[ri][jj]);
                            }
                    }
                };
                st_rows_load(0);
                umma::wg_wait<0>();
                __syncthreads();
                if (mine) {
#pragma unroll
                    for (int j = 0; j < 8; j++)
#pragma unroll
                        for (int p = 0; p < 2; p++)
#pragma unroll
                            for (int e = 0; e < 2; e++) {
                                const int idx = umma::tile_index2(8 * j + 2 * t4 + e, p ? rB : rA, 64, TL), c = 4 * j + 2 * p + e;
                                arena[AR_A_HI / 4 + idx] = dz1[c]; arena[AR_A_LO / 4 + idx] = tf32_lo(dz1[c]);   // dZ1^T
                            }
                }
                st_rows_scatter(0);
                st_rows_load(4);
                st_rows_scatter(4);
                umma::fence_async_smem();
                __syncthreads();
                if (n_dw1) gemm3_n(n_dw1, g2, TA_hi, TA_lo, TB_hi.rows_from(64 * h), TB_lo.rows_from(64 * h), !first);
                if (h == 1) umma::gemm3<32>(g1 + 16, TA_hi, TA_lo, TE, TE, 64, !first, false, true);
                umma::wg_commit();
                umma::wg_wait<0>();
            }
            umma::fence_async_smem();   // the arena was written through the generic proxy, the next W1 copy is a TMA write
            __syncthreads();            // the arena is free: the next tile's W1 copy / the gradient staging may overwrite it
        }

        TC_STAMP(8);
        // ================= AdamW ==========
        // column sums of dW3 over the warp's rows: lanes with equal lane % 4 hold the same columns
#pragma unroll
        for (int c = 0; c < 16; c++) {
            float v = dw3[c];
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 8);
            v += __shfl_xor_sync(0xffffffffu, v, 16);
            if (lane < 4) mi.redw[warp][8 * (c >> 1) + 2 * lane + (c & 1)] = v;
        }
        {
            const float ms = warp_sum(mae_acc), ds = warp_sum(db3_acc);
            if (lane == 0) { mi.redmae[warp] = ms; mi.reddb3[warp] = ds; }
        }
        {
            // 1) gradients registers -> shared staging in region 2 (the arena is free)
            float *gs_w2 = reinterpret_cast<float *>(smem + REG2);     // [64][65]
            const int pitch1 = d.D | 1;
            float *gs_w1 = gs_w2 + 64 * 65;                            // [64][pitch1]   (state cols, then action cols)
            float *gs_b1 = gs_w1 + 64 * pitch1, *gs_b2 = gs_b1 + 64;
#pragma unroll
            for (int p = 0; p < 2; p++) {
                const int j = p ? rB : rA;                             // the gradient's row = hidden unit
#pragma unroll
                for (int jb = 0; jb < 8; jb++)
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const int c = 8 * jb + 2 * t4 + e, k = 64 * h + c;
                        if (h == 0) gs_w2[j * 65 + c] = g1[4 * jb + 2 * p + e];
                        if (c < n_dw1 && k < d.obs) gs_w1[j * pitch1 + k] = g2[4 * jb + 2 * p + e];
                        if (h == 1 && jb < 4) {                        // [db | dW1a] columns: 0 = bias, 1 + k = action k
                            if (c == 0) { gs_b2[j] = g1[4 * jb + 2 * p + e]; gs_b1[j] = g1[16 + 4 * jb + 2 * p + e]; }
                            else if (c - 1 < d.A) gs_w1[j * pitch1 + d.obs + c - 1] = g1[16 + 4 * jb + 2 * p + e];
                        }
                    }
            }
            __syncthreads();
            // 2) AdamW over the flat parameter vector, all 256 threads, fully coalesced 16-byte accesses.  The sweep is bound by
            //    L2 round trips, not bytes: W1 | W2 are walked as ONE flat list of 16-byte groups (no 4-lane tail passes per W1
            //    row) in batches of two groups per thread whose 8 loads are issued before the first use, and the loads of the
            //    small vectors (b1 | b2 | W3 | b3, one parameter per thread) are in flight across the whole sweep.
            const float2 sc = L.scal[round];
            AdamScalarsTc hs;
            hs.decay = a.decay; hs.omb1 = a.omb1; hs.beta2 = a.beta2; hs.omb2 = a.omb2; hs.eps = a.eps;
            hs.step_size = sc.x; hs.bc2_sqrt = sc.y; hs.inv_bc2_sqrt = 1.0f / sc.y;
            int si = -1;                // this thread's small parameter
            float sg = 0.f, sw = 0.f, sm = 0.f, sv2 = 0.f, sx = 0.f;
            if (tid < 64) { si = d.ob1 + tid; sg = gs_b1[tid]; }
            else if (tid < 128) { si = d.ob2 + tid - 64; sg = gs_b2[tid - 64]; }
            else if (tid < 192) {       // W3: sum the eight warps' partials of this column in fixed order
                const int col = tid - 128;
                sg = 0.f;
#pragma unroll
                for (int w8 = 0; w8 < 8; w8++) sg += mi.redw[w8][col];
                si = d.oW3 + col;
            } else if (tid == 192) {
                float e = 0.f;
#pragma unroll
                for (int w8 = 0; w8 < 8; w8++) { sg += mi.reddb3[w8]; e += mi.redmae[w8]; }
                si = d.ob3;
                L.out_mae[round] = e / (float)a.B;   // reported "loss": mean |q - y|
            }
            if (si >= 0) { sw = __ldcg(L.w + si); sm = __ldcg(L.m + si); sv2 = __ldcg(L.v + si); sx = __ldcg(L.vmax + si); }
            const bool vecD = ((d.D & 3) == 0) && ((d.oW2 & 3) == 0);
            if (vecD) {
                constexpr int U = 2;
                const int D4 = d.D >> 2, n1 = HID * D4, ntot = n1 + HID * HID / 4;
                for (int q0 = tid; q0 < ntot; q0 += U * NTH) {
                    float4 w4[U], m4[U], v4[U], x4[U];
#pragma unroll
                    for (int u = 0; u < U; u++) {
                        const int q = q0 + u * NTH;
                        if (q < ntot) {
                            const int i = q < n1 ? d.oW1 + q * 4 : d.oW2 + (q - n1) * 4;   // W1 rows are contiguous: row * D + c4 * 4 == q * 4
                            w4[u] = __ldcg(reinterpret_cast<const float4 *>(L.w + i)); m4[u] = __ldcg(reinterpret_cast<const float4 *>(L.m + i));
                            v4[u] = __ldcg(reinterpret_cast<const float4 *>(L.v + i)); x4[u] = __ldcg(reinterpret_cast<const float4 *>(L.vmax + i));
                        }
                    }
#pragma unroll
                    for (int u = 0; u < U; u++) {
                        const int q = q0 + u * NTH;
                        if (q < ntot) {
                            const bool is_w1 = q < n1;
                            int i, row, c;
                            const float *gp;
                            if (is_w1) {
                                row = q / D4; c = (q - row * D4) * 4;
                                i = d.oW1 + q * 4;
                                gp = gs_w1 + row * pitch1 + c;
                            } else {
                                const int q4 = q - n1;
                                row = q4 >> 4; c = (q4 & 15) * 4;
                                i = d.oW2 + q4 * 4;
                                gp = gs_w2 + row * 65 + c;
                            }
                            float4 w = w4[u], mm = m4[u], vv = v4[u], xx = x4[u];
                            w.x = adam_math(w.x, mm.x, vv.x, xx.x, gp[0], hs); w.y = adam_math(w.y, mm.y, vv.y, xx.y, gp[1], hs);
                            w.z = adam_math(w.z, mm.z, vv.z, xx.z, gp[2], hs); w.w = adam_math(w.w, mm.w, vv.w, xx.w, gp[3], hs);
                            *reinterpret_cast<float4 *>(L.w + i) = w; *reinterpret_cast<float4 *>(L.m + i) = mm;
                            *reinterpret_cast<float4 *>(L.v + i) = vv; *reinterpret_cast<float4 *>(L.vmax + i) = xx;
                            // the same values in the operand-layout tiles (hi = the value, lo = residual)
                            if (is_w1) {
                                if (c < d.obs) {
                                    const int ti = umma::tile_index(row, c, d.obs);
                                    *reinterpret_cast<float4 *>(To.w1hi + ti) = w;
                                    *reinterpret_cast<float4 *>(To.w1lo + ti) = make_float4(tf32_lo(w.x), tf32_lo(w.y), tf32_lo(w.z), tf32_lo(w.w));
                                }
                            } else {   // kperm order: columns c, c + 2 and c + 1, c + 3 are neighbours
                                const int te = umma::tile_index(row, umma::kperm(c), HID), to = umma::tile_index(row, umma::kperm(c + 1), HID);
                                *reinterpret_cast<float2 *>(To.w2 + te) = make_float2(w.x, w.z);
                                *reinterpret_cast<float2 *>(To.w2 + to) = make_float2(w.y, w.w);
                                *reinterpret_cast<float2 *>(To.w2 + 4096 + te) = make_float2(tf32_lo(w.x), tf32_lo(w.z));
                                *reinterpret_cast<float2 *>(To.w2 + 4096 + to) = make_float2(tf32_lo(w.y), tf32_lo(w.w));
                            }
                        }
                    }
                }
            } else {
                for (int row = warp; row < HID; row += 8)
                    for (int c = lane; c < d.D; c += 32) {
                        const int i = d.oW1 + row * d.D + c;
                        float mm = __ldcg(L.m + i), vv = __ldcg(L.v + i), xx = __ldcg(L.vmax + i);
                        L.w[i] = adam_math(__ldcg(L.w + i), mm, vv, xx, gs_w1[row * pitch1 + c], hs);
                        L.m[i] = mm; L.v[i] = vv; L.vmax[i] = xx;
                    }
                for (int e = tid; e < HID * HID; e += NTH) {
                    const int i = d.oW2 + e;
                    float mm = __ldcg(L.m + i), vv = __ldcg(L.v + i), xx = __ldcg(L.vmax + i);
                    L.w[i] = adam_math(__ldcg(L.w + i), mm, vv, xx, gs_w2[(e >> 6) * 65 + (e & 63)], hs);
                    L.m[i] = mm; L.v[i] = vv; L.vmax[i] = xx;
                }
                __syncthreads();
                rebuild_tiles(L.w, d, To, tid);         // unaligned shapes (D % 4 != 0): tiles from the flat vector
            }
            fence_proxy_async_all();                    // the tile writes are read by TMA in the next round
            if (si >= 0) {
                L.w[si] = adam_math(sw, sm, sv2, sx, sg, hs);
                L.m[si] = sm; L.v[si] = sv2; L.vmax[si] = sx;
            }
        }
        __syncthreads();
        TC_STAMP(9);
    }
}

// a few microseconds of nothing: lets the learner CTAs of the main stream take their SMs before the next chunk's
// index producers (side stream) become ready
__global__ void k_delay(unsigned ns) {
    const long long t0 = clock64();
    while (clock64() - t0 < (long long)ns * 2) __nanosleep(200);
}

// all learners' index streams in one launch: CTA i draws `rounds` samples for learner i
struct MultiSampler {
    uint32_t *mt_state;
    SamplerParams sp;
};
__global__ void __launch_bounds__(kSamplerThreads, 1) k_sample_indices_multi(const MultiSampler *items, int rounds, int round0) {
    extern __shared__ __align__(16) unsigned char dyn[];
    __shared__ SamplerState S;
    MultiSampler it = items[blockIdx.x];
    if (it.sp.out_slot) it.sp.out_slot += (size_t)round0 * it.sp.k;
    if (it.sp.out_logical) it.sp.out_logical += (size_t)round0 * it.sp.k;
    sampler_init(S, it.mt_state, dyn, it.sp);
    sampler_advance(S, dyn, it.sp, rounds);
    __syncthreads();
    sampler_store(S, it.mt_state);
}

}  // namespace

static bool tc_eligible(const prl_dqn_cfg &c, int batch) {
    const bool a_ok = c.n_actions == 1 || c.n_actions == 2 || c.n_actions == 4 || c.n_actions == 8 || c.n_actions == 16;
    return c.hidden1 == HID && c.hidden2 == HID && c.obs_dim % 8 == 0 && c.obs_dim >= 8 && c.obs_dim <= 128 && a_ok &&
           !c.double_dqn && (batch == 128 || batch == 256);
}

extern "C" int prl_dqn_tc_supported(const prl_dqn *q, int batch) { return q && q->tc_tiles && tc_eligible(q->cfg, batch) ? 1 : 0; }

extern "C" int prl_dqn_learn_multi(prl_dqn *const *dqns, prl_buf *const *bufs, int count, int rounds, int batch,
                                   const int64_t *training_steps0, float *const *out_mae, float *const *out_q,
                                   float *const *out_y, int32_t *const *out_logical, void *stream_) {
    PRL_REQUIRE(dqns && bufs && training_steps0 && out_mae && count > 0, "null / empty argument");
    cudaStream_t stream = (cudaStream_t)stream_;
    prl_dqn *q0 = dqns[0];
    const prl_dqn_cfg &c = q0->cfg;
    if (!tc_eligible(c, batch))
        return fail(PRL_EUNSUPPORTED,
                    "tensor-core learner needs hidden [64,64], obs %% 8 == 0 <= 128, actions in {1,2,4,8,16}, DQN, batch 128/256");
    PRL_REQUIRE(rounds > 0 && rounds <= c.max_rounds && batch <= c.max_batch, "rounds / batch outside the configured maxima");
    PRL_REQUIRE((size_t)count * (sizeof(TcLearner) + sizeof(MultiSampler)) <= 64 * 1024, "too many learners in one group");
    PRL_REQUIRE(count <= q0->sm_count, "more learners than SMs in one launch");
    // per-learner descriptors are staged in pinned memory of learner 0 and copied to its workspace
    static thread_local TcLearner *h_learn = nullptr;
    static thread_local MultiSampler *h_samp = nullptr;
    static thread_local cudaEvent_t h_done = nullptr;
    if (!h_learn) {
        PRL_CUDA(cudaHostAlloc((void **)&h_learn, 32 * 1024, cudaHostAllocDefault));
        PRL_CUDA(cudaHostAlloc((void **)&h_samp, 32 * 1024, cudaHostAllocDefault));
        PRL_CUDA(cudaEventCreateWithFlags(&h_done, cudaEventDisableTiming));
    }
    PRL_CUDA(cudaEventSynchronize(h_done));
    size_t samp_smem = 0;
    for (int i = 0; i < count; i++) {
        prl_dqn *q = dqns[i];
        prl_buf *b = bufs[i];
        PRL_REQUIRE(q && b, "null learner / buffer");
        const prl_dqn_cfg &ci = q->cfg;
        PRL_REQUIRE(ci.obs_dim == c.obs_dim && ci.n_actions == c.n_actions && ci.hidden1 == c.hidden1 &&
                        ci.hidden2 == c.hidden2 && ci.double_dqn == c.double_dqn &&
                        ci.target_update_freq == c.target_update_freq && ci.lr == c.lr && ci.beta1 == c.beta1 &&
                        ci.beta2 == c.beta2 && ci.eps == c.eps && ci.weight_decay == c.weight_decay &&
                        ci.gamma == c.gamma && ci.tau == c.tau && rounds <= ci.max_rounds && batch <= ci.max_batch,
                    "all learners of a group must share one configuration");
        PRL_REQUIRE(q->tc_tiles, "learner %d has no operand-tile workspace", i);
        PRL_REQUIRE((b->desc.flags & PRL_BUF_DISCRETE) && b->desc.obs_dim == c.obs_dim && b->desc.n_actions == c.n_actions,
                    "buffer %d does not match the learner", i);
        PRL_REQUIRE(b->lay.record_words == bufs[0]->lay.record_words && b->lay.off_avail == bufs[0]->lay.off_avail,
                    "buffers must share one record layout");
        // the per-round AdamW scalars (two double pow() per round, as torch evaluates them) depend only on the shared
        // configuration and the step count: learners at the same step read learner 0's copy
        const bool shared_scal = i > 0 && q->adam_step == q0->adam_step;
        int rc = shared_scal ? PRL_OK : prl_dqn_stage_scalars(q, rounds, stream);
        if (rc) return rc;
        size_t sbytes = 0;
        rc = prl_sampler_params(b, batch, &h_samp[i].sp, &sbytes);
        if (rc) return rc;
        if (sbytes > samp_smem) samp_smem = sbytes;
        h_samp[i].mt_state = b->mt_state;
        h_samp[i].sp.out_slot = q->slots;
        h_samp[i].sp.out_logical = out_logical ? out_logical[i] : nullptr;
        TcLearner &L = h_learn[i];
        L.records = b->records; L.slots = q->slots;
        L.tiles = q->tc_tiles;
        L.w = q->w; L.wt = q->wt; L.m = q->m; L.v = q->v; L.vmax = q->vmax;
        L.scal = shared_scal ? q0->scal_dev : q->scal_dev;
        L.out_mae = out_mae[i]; L.out_q = out_q ? out_q[i] : nullptr; L.out_y = out_y ? out_y[i] : nullptr;
        L.steps0 = training_steps0[i];
        L.buf_flags = b->desc.flags;
        L.pad_ = 0;
    }
    TcLearner *d_learn = reinterpret_cast<TcLearner *>(q0->multi_dev);
    MultiSampler *d_samp = reinterpret_cast<MultiSampler *>(reinterpret_cast<char *>(q0->multi_dev) + 32 * 1024);
    PRL_CUDA(cudaMemcpyAsync(d_learn, h_learn, (size_t)count * sizeof(TcLearner), cudaMemcpyHostToDevice, stream));
    PRL_CUDA(cudaMemcpyAsync(d_samp, h_samp, (size_t)count * sizeof(MultiSampler), cudaMemcpyHostToDevice, stream));
    PRL_CUDA(cudaEventRecord(h_done, stream));

    PRL_CUDA(cudaFuncSetAttribute(k_sample_indices_multi, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));

    TcArgs a;
    a.learners = d_learn;
    a.lay = bufs[0]->lay;
    a.d = q0->d;
    a.B = batch; a.rounds = rounds; a.freq = c.target_update_freq; a.round0 = 0;
    a.decay = (float)(1.0 - c.lr * c.weight_decay);
    a.omb1 = (float)(1.0 - c.beta1);
    a.beta2 = (float)c.beta2;
    a.omb2 = (float)(1.0 - c.beta2);
    a.eps = (float)c.eps;
    a.gamma = (float)c.gamma;
    a.tau = (float)c.tau;
    a.omtau = (float)(1.0 - c.tau);
    a.inv_b2 = 2.0f / (float)batch;
    a.prof = q0->prof;
    { static const int c = [] { const char *e = getenv("PRL_TC_PROF_CTA"); return e ? atoi(e) : 0; }(); a.prof_cta = c; }
    const size_t smem = MISC_OFF + sizeof(Misc);
    PRL_REQUIRE(smem <= (size_t)q0->max_smem, "tensor-core learner needs %zu B of shared memory", smem);
    PRL_CUDA(cudaFuncSetAttribute(k_dqn_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));

    // The index streams are produced in chunks of rounds: chunk 0 ahead of the first learner launch, chunk c + 1 on a
    // side stream WHILE the learners run chunk c (one learner CTA fills an SM, so the producers of the next chunk run
    // on the SMs the group leaves free; with no spare SM they simply run between the learner launches).
    const int spare = q0->sm_count - count;
    int nchunks = 1;
    if (!q0->prof && spare >= 2 && rounds >= 64) nchunks = rounds >= 256 ? 4 : 2;
    static thread_local cudaStream_t side = nullptr;
    static thread_local cudaEvent_t ev_idx[8], ev_fork = nullptr;
    if (nchunks > 1 && !side) {
        PRL_CUDA(cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking));
        for (auto &e : ev_idx) PRL_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        PRL_CUDA(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
    }
    // chunk 0 is the only one whose index production is NOT hidden behind a learner launch: keep it short (32 rounds)
    const int first = nchunks > 1 ? (rounds / nchunks < 32 ? rounds / nchunks : 32) : rounds;
    auto chunk_begin = [&](int cix) {
        return cix == 0 ? 0 : first + (int)((long long)(rounds - first) * (cix - 1) / (nchunks > 1 ? nchunks - 1 : 1));
    };
    k_sample_indices_multi<<<count, kSamplerThreads, samp_smem, stream>>>(d_samp, chunk_begin(1), 0);
    PRL_CUDA(cudaGetLastError());
    if (nchunks > 1) {
        PRL_CUDA(cudaEventRecord(ev_fork, stream));
        PRL_CUDA(cudaStreamWaitEvent(side, ev_fork, 0));
    }
    if (q0->timing) PRL_CUDA(cudaEventRecord(q0->t0, stream));
    for (int cix = 0; cix < nchunks; cix++) {
        const int r0 = chunk_begin(cix), r1 = chunk_begin(cix + 1);
        if (cix > 0) PRL_CUDA(cudaStreamWaitEvent(stream, ev_idx[cix], 0));
        a.round0 = r0; a.rounds = r1 - r0;
        k_dqn_tc<<<count, NTH, smem, stream>>>(a);
        PRL_CUDA(cudaGetLastError());
        if (cix + 1 < nchunks) {
            const int n0 = r1, n1 = chunk_begin(cix + 2);
            k_delay<<<1, 1, 0, side>>>(30000u);
            k_sample_indices_multi<<<count, kSamplerThreads, samp_smem, side>>>(d_samp, n1 - n0, n0);
            PRL_CUDA(cudaGetLastError());
            PRL_CUDA(cudaEventRecord(ev_idx[cix + 1], side));
        }
    }
    if (q0->timing) PRL_CUDA(cudaEventRecord(q0->t1, stream));
    for (int i = 0; i < count; i++) {
        dqns[i]->adam_step += rounds;
        dqns[i]->last_launches = 3 * nchunks - 1;   // index producers + learner launches + the side-stream delays
        dqns[i]->last_ctas = 1;
        dqns[i]->last_rows = batch;
    }
    return PRL_OK;
}
