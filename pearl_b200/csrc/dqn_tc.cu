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
//   layer 1  T1 = X W1s^T: the rows are gathered into shared memory by cp.async (K chunks of 64, double-buffered, the
//            first chunk issued ahead of time) and read back as register A fragments (RS form); B = the W1 tile.
//   phase T  target net: per action slot one 64 x 64 x 64 product whose A operand relu(T1 + W1a[:,a] + b1) is
//            built in registers from the layer-1 accumulator and never leaves them; running max over the slots.
//   phase O  online net forward the same way, loss gradient, dZ2, dH1 = dZ2 W2 (B operand = W2^T tile), all on
//            register operands; then the weight gradients as products over the batch dimension:
//            dW2 = dZ2^T H1, dW1s = dZ1^T S, and [db | dW1a] = dZ^T E with E = [1 | onehot(action)];
//            their operands are explicitly transposed tiles written with a 144-byte chunk pitch
//            (bank-conflict-free column scatter), 64 batch rows per pass, the two warpgroups issuing the same
//            products on equal shares of the output columns.  The warpgroup that owns the pass's rows scatters their
//            dZ2^T, H1^T and dZ1^T, the other one E^T.  For obs > 64 dW1s is computed as its transpose S^T dZ1, whose A
//            operand S^T is read as register fragments straight out of layer 1's staging buffers (warpgroup h takes
//            obs rows [64 h, 64 h + 64), its K chunk h) and whose B operand is the dZ1^T tile; for obs <= 64 both
//            warpgroups scatter S^T from state rows re-read from global memory.  The accumulators stay in registers
//            for the whole step.
//   AdamW    gradients registers -> shared staging, then one sweep over the flat W1 | b1 | W2 range whose parameters and
//            moments stream in by TMA bulk copies, in 16 KB chunks through an 8-slot ring in regions 3 and 1 (free once
//            the last weight-gradient products have been waited for); 16-byte stores write the results, and the new W1 | W2
//            replace their gradients in the staging, from which a second pass writes the operand-layout weight tiles in
//            tile order (coalesced).  b1 | b2 | W3 | b3 are updated one parameter per thread.  Shapes with
//            D % 4 != 0 (1 or 2 actions) or parameters that are not 16-byte aligned take a scalar sweep instead.
//
// The weights are kept in global memory a second time IN THE OPERAND LAYOUT (hi tile = the fp32 values — the tensor
// core truncates them to TF32 — and lo tile = x - trunc_tf32(x)), written by AdamW / the soft target update next to the
// flat torch-order vectors, so staging a network's B operands is three TMA bulk copies (cp.async.bulk + mbarrier
// complete_tx) issued by one thread.  The W2 and W2^T tiles store their K axis in the order umma::kperm, which is the
// order in which an accumulator's columns feed the next product's register A operand.  The online network's tiles are
// fetched once per row tile: the weight-gradient passes use regions 1 and 3 for their transposed tiles and for dZ1,
// which waits there for its pass.  The target network's small vectors are
// cached in shared memory between soft updates, the soft target update is applied to the tiles in tile order.
//
// Each 3xTF32 product is one chain of wgmma with a single wait at its end, and that only holds while ptxas can pipeline
// the kernel's wgmma: ONE obstacle anywhere in the kernel makes it wait after every wgmma of the kernel.  What must
// stay true: no function call in the kernel (not even printf, C7510); no wgmma under
// a branch, including a runtime step count or a branch on the warpgroup index (both warpgroups issue the same products,
// C7520), and no conditional load feeding an A fragment; and each chain fits in the registers together with everything
// live across it (C7511 / C7512), which is why H1 and dZ2 wait in shared memory while dH1 is formed, dZ1 until its
// weight-gradient pass, and the learner descriptor and the dW3 partial sums live in shared memory.  For the same reason
// the phase stamps (TC_STAMP) are predicated stores rather than branches.  tests/test_dqn_tc_sass.py checks the SASS.
// Spills cost more here than usual: the 225 KB of shared memory leave at most 28 KB of L1 for the spill frame of 256
// threads, so spill traffic reaches L2.  Values that are the same in every round must not be hoisted out of the round
// loop into registers: the wgmma descriptors are built next to each wgmma (umma::Tile::desc) and the shared-memory
// offsets that follow from the thread index are recomputed where they are used (tid_here).  Hoisted, both stay live
// across every chain and make up most of the spills.  tests/test_dqn_tc_spills.py bounds the spill bytes and keeps
// spill reloads out of the chains.
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
// transposed-tile arena for the weight-gradient products, 64 batch rows per pass: TA hi | lo, TE and TB lo in region 1,
// TB hi in the W2^T half of region 3 (both re-fetched for the next row tile).  Region 2 is left alone: the state rows
// that layer 1 staged there are the S^T operand of dW1s.
constexpr int TL = 144;              // chunk pitch of transposed tiles
constexpr int AR_A_HI = 0, AR_A_LO = 18432, AR_E = 36864, AR_B_LO = 46080, AR_B_HI = REG3 + HALF;
// AdamW ring: chunks of ACH flat parameters, one slot = the chunk's w | m | v | vmax (16 KB); slots 0-3 in region 3,
// 4-7 in region 1
constexpr int ACH = 1024, ARING = 8, ASLOT = 4 * ACH * 4;

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
    int adam_tma;      // D % 4 == 0 and every learner's w / m / v / vmax 16-byte aligned: AdamW streams them by TMA
};

// A predicated store, not a branch: a stamp under `if` between two products costs the registers the chains need
__device__ __forceinline__ void tc_stamp(const TcArgs &a, int round, int idx) {
    long long *p = a.prof + (size_t)round * 16 + idx;
    const unsigned on = (a.prof != nullptr) & (blockIdx.x == (unsigned)a.prof_cta) & (threadIdx.x == 0);
    asm volatile("{\n\t.reg .pred q;\n\t.reg .u64 c;\n\tsetp.ne.u32 q, %1, 0;\n\tmov.u64 c, %%clock64;\n\t@q st.global.u64 [%0], c;\n\t}"
                 ::"l"(p), "r"(on) : "memory");
}
#define TC_STAMP(idx) tc_stamp(a, round, (idx))

struct Misc {
    // small fp32 vectors of a network: W1[:, obs + a] + b1, b2, w3, b3.  [0] online, [1] target (the target's only change at
    // a scheduled soft update, so they are loaded then and in the prologue, not every round)
    struct Smalls { float watb[16][HID]; float b2[HID], w3[HID]; float b3, pad0[3]; } sm[2];
    float y[MAX_B];
    int act[MAX_B], cnt[MAX_B], slot[MAX_B];
    float rew[MAX_B], term[MAX_B];
    float redw[8][HID];
    float redmae[8], reddb3[8];
    unsigned long long bar[3 + ARING];   // 0: target tiles; 1: online W1 tiles; 2: online W2 | W2^T tiles; 3 + s: AdamW ring slot s
    // kept here rather than in registers: the wgmma chains need the registers (section 3.1 of DESIGN.md)
    TcLearner L;                 // this CTA's learner, per-round arrays shifted to the launch's first round
    float dw3[16][NTH];          // per-thread dW3 partial sums, carried across the row tiles
};

__device__ __forceinline__ void cp_async16_zfill_tc(void *smem_dst, const void *gmem_src, int src_bytes) {
    unsigned sa = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(sa), "l"(gmem_src), "r"(src_bytes) : "memory");
}

// threadIdx.x, opaque to the compiler at the point of use: the shared-memory offsets derived from it are recomputed where
// they are needed instead of being hoisted out of the round loop and kept live (and spilled) across the wgmma chains
__device__ __forceinline__ int tid_here() {
    int t = threadIdx.x;
    asm volatile("" : "+r"(t));
    return t;
}
// this thread's row p (0, 1) of its warpgroup's 64-row block (umma::acc_row), from tid_here()
__device__ __forceinline__ int acc_row_here(int p) {
    const int t = tid_here();
    return ((t >> 5) & 3) * 16 + ((t & 31) >> 2) + 8 * p;
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
//   [W1 hi: 64 x k1][W1 lo][W2 hi: 64 x 64][W2 lo]      (the shared-memory images, tile by tile; the W2 tiles with their
//   K axis in umma::kperm order)
// and for the online network then [W2^T hi: 64 x 64][W2^T lo], the B operand of dH1 = dZ2 W2 (contraction over W2's rows),
// with its K axis in kperm order too.  The target network needs no W2^T.
// The W1 tiles have K = k1 = obs rounded up to a multiple of 64, the columns from obs on are zero: every layer-1 K chunk is
// a full 8-step product (no runtime step count inside a wgmma chain), and the padding adds exact zeros to the sums.
struct NetTiles { float *w1hi, *w1lo, *w2, *w2t; };   // w2 / w2t: 2 x 4096-float blocks hi | lo; w2t null for the target
__host__ __device__ inline int k1_cols(int obs) { return (obs + 63) & ~63; }
__host__ __device__ inline int net_tile_floats(int obs) { return 128 * k1_cols(obs) + 2 * HID * HID; }   // without W2^T
__device__ __forceinline__ NetTiles net_tiles(float *base, int obs, bool with_w2t) {
    const int k1 = k1_cols(obs), n = net_tile_floats(obs);
    return NetTiles{base, base + 64 * k1, base + 128 * k1, with_w2t ? base + n : nullptr};
}
// all tiles of one network from its flat parameter vector (kernel prologue, scalar AdamW sweep)
__device__ void rebuild_tiles(const float *__restrict__ net, const Dims &d, const NetTiles &t, int tid) {
    const int k1 = k1_cols(d.obs);
    for (int e = tid; e < HID * k1; e += NTH) {
        const int j = e / k1, k = e - j * k1;
        const float x = k < d.obs ? __ldcg(net + d.oW1 + (size_t)j * d.D + k) : 0.f;
        const int idx = umma::tile_index(j, k, k1);
        t.w1hi[idx] = x; t.w1lo[idx] = tf32_lo(x);
    }
    for (int e = tid; e < HID * HID; e += NTH) {
        const int j = e >> 6, k = e & 63;
        const float x = __ldcg(net + d.oW2 + e);
        const int i1 = umma::tile_index(j, umma::kperm(k), HID);
        t.w2[i1] = x; t.w2[4096 + i1] = tf32_lo(x);
        if (t.w2t) {
            const int i2 = umma::tile_index(k, umma::kperm(j), HID);
            t.w2t[i2] = x; t.w2t[4096 + i2] = tf32_lo(x);
        }
    }
}
// the small fp32 vectors of a network (action columns + b1, b2, w3, b3); all loads of a thread issued before the first use
__device__ void load_smalls(const float *__restrict__ net, const Dims &d, Misc::Smalls &mi) {
    const int tid = tid_here();
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
// arrive by coalesced 16-byte cp.async (16 lanes per row) in staging buffers [64 rows][64 floats] whose 16-byte chunk c
// of row r sits at chunk position c ^ (r & 7), which makes the fragment reads below (8 rows x 4 consecutive k per warp
// and load) conflict free; 64 columns of K per chunk.  Each warpgroup has two buffers, K chunk kc goes to buffer kc & 1:
// chunk kc + 1 is in flight while chunk kc is multiplied, and chunk 0 of a block is issued by the caller (l1_issue)
// ahead of layer1_block, as early as its buffer is free.
__device__ __forceinline__ void l1_issue(const TcArgs &a, const TcLearner &L, const Misc &mi, char *smem, int field_off, int row0, int kc) {
    const int ft = tid_here(), m = ft & 127, g = ft >> 7;
    float *sbuf = reinterpret_cast<float *>(smem + REG2 + g * 2 * SBUF + (kc & 1) * SBUF);
#pragma unroll 4
    for (int i = 0; i < 8; i++) {
        const int item = i * 128 + m, rr = item >> 4, c = item & 15, k = kc * 64 + c * 4;
        const float *src = reinterpret_cast<const float *>(L.records + (size_t)mi.slot[row0 + rr] * a.lay.record_words) + field_off + k;
        const int nb = k < a.d.obs ? 16 : 0;
        cp_async16_zfill_tc(sbuf + rr * 64 + ((c ^ (rr & 7)) << 2), nb ? src : reinterpret_cast<const float *>(L.records), nb);
    }
    cp_async_commit();
}
__device__ __forceinline__ void layer1_block(const TcArgs &a, const TcLearner &L, const Misc &mi, char *smem, int field_off, int row0,
                                             float (&t1)[32]) {
    const int g = threadIdx.x >> 7;
    const int k1 = k1_cols(a.d.obs);
    const umma::Tile B_hi = umma::make_tile(smem + REG1, k1, 128), B_lo = umma::make_tile(smem + REG1 + HALF, k1, 128);
    for (int kc = 0; kc * 64 < k1; kc++) {
        if ((kc + 1) * 64 < k1) l1_issue(a, L, mi, smem, field_off, row0, kc + 1);
        else cp_async_commit();          // empty group: the wait below always leaves exactly the newest group in flight
        cp_async_wait<1>();
        group_sync(g);
        const float *sbuf = reinterpret_cast<const float *>(smem + REG2 + g * 2 * SBUF + (kc & 1) * SBUF);
        const int t = tid_here() & 3, r0 = acc_row_here(0);
        float hi[32], lo[32];
#pragma unroll
        for (int ks = 0; ks < 8; ks++)
#pragma unroll
            for (int q = 0; q < 2; q++)
#pragma unroll
                for (int p = 0; p < 2; p++) {
                    const int r = r0 + 8 * p, k = 8 * ks + t + 4 * q;
                    umma::split_tf32(sbuf[r * 64 + (((k >> 2) ^ (r & 7)) << 2) + (k & 3)], hi[4 * ks + 2 * q + p], lo[4 * ks + 2 * q + p]);
                }
        group_sync(g);   // the buffer is free for chunk kc + 2 (or chunk 0 of the next block)
        umma::gemm3_rs<HID, 8>(t1, hi, lo, B_hi.shifted(kc * 2048), B_lo.shifted(kc * 2048), kc > 0);
        umma::wg_commit();
        umma::wg_wait<0>();
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

// A shared-memory load the compiler may not hoist out of a loop: the small vectors (w3, b2, ...) are the same in every
// action slot / row tile, and keeping them in registers across the loop costs the registers the wgmma chains need.
__device__ __forceinline__ float2 lds2(const float *p) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(umma::smem_u32(p)));
    return v;
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

// dW1s columns per warpgroup: the two warpgroups take equal shares [0, NW) and [NW, 2 NW) of the obs columns
__host__ __device__ inline int dw1_share(int obs) { return obs > 64 ? 64 : obs > 32 ? 32 : obs > 16 ? 16 : 8; }

__device__ const uint8_t kIota[16] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15};

template <int NW>
__global__ void __launch_bounds__(NTH, 1) k_dqn_tc(const TcArgs a) {
    extern __shared__ __align__(1024) char smem[];
    Misc &mi = *reinterpret_cast<Misc *>(smem + MISC_OFF);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        TcLearner L = a.learners[blockIdx.x];
        if (a.round0) {   // a later chunk of the same call: shift every per-round array once
            L.slots += (size_t)a.round0 * a.B;
            L.scal += a.round0;
            L.out_mae += a.round0;
            if (L.out_q) L.out_q += (size_t)a.round0 * a.B;
            if (L.out_y) L.out_y += (size_t)a.round0 * a.B;
            L.steps0 += a.round0;
        }
        mi.L = L;
    }
    __syncthreads();
    const TcLearner &L = mi.L;
    const Dims &d = a.d;
    const int h = tid >> 7, t4 = tid & 3;
    const int ntiles = a.B >> 7;
    const int W = a.lay.record_words;

    // De-phase the learners: identical CTAs started together run in lock-step and hit L2 / HBM with their AdamW sweeps
    // (432 KB each) and row gathers all at once; a start offset of up to ~50 us spreads those bursts over the round.
    if (tid == 0 && gridDim.x > 1) {
        const long long t0 = clock64(), wait = (long long)(blockIdx.x % 48) * 2000;
        while (clock64() - t0 < wait) __nanosleep(100);
    }
    uint64_t *bar = reinterpret_cast<uint64_t *>(mi.bar);
    if (tid == 0)
        for (int i = 0; i < 3 + ARING; i++) umma::mbar_init(bar + i, 1);
    // the operand-layout tiles follow the flat parameters (which the host may have changed between calls)
    auto To = [&] { return net_tiles(L.tiles, d.obs, true); };
    auto Tt = [&] { return net_tiles(L.tiles + net_tile_floats(d.obs) + 2 * HID * HID, d.obs, false); };
    rebuild_tiles(L.w, d, To(), tid);
    rebuild_tiles(L.wt, d, Tt(), tid);
    fence_proxy_async_all();
    __syncthreads();
    const int k1 = k1_cols(d.obs);
    const uint32_t w1_bytes = 64u * k1 * 4, w2_bytes = 2u * HID * HID * 4;
    // target tiles: three TMA bulk copies, W1 hi / lo into region 1 and W2 hi | lo into region 3
    auto tma_target = [&] {
        mbar_expect_tx(bar + 0, 2 * w1_bytes + w2_bytes);
        bulk_g2s(smem + REG1, Tt().w1hi, w1_bytes, bar + 0);
        bulk_g2s(smem + REG1 + HALF, Tt().w1lo, w1_bytes, bar + 0);
        bulk_g2s(smem + REG3, Tt().w2, w2_bytes, bar + 0);
    };
    // B-operand tiles of the online network by TMA, once per row tile (the weight-gradient passes overwrite them): W1 hi / lo
    // into region 1 on bar[1], the W2 and W2^T blocks (adjacent in global memory) into region 3 on bar[2].  Two barriers, so
    // that layer 1 waits for W1 only and W2 | W2^T keep loading under it.  (Issuing row tile 0's W1 inside phase T, after
    // the last target layer 1, together with this later wait made ptxas serialise every wgmma of the NW = 64 kernel, C7520.)
    auto tma_online_w1 = [&] {
        mbar_expect_tx(bar + 1, 2 * w1_bytes);
        bulk_g2s(smem + REG1, To().w1hi, w1_bytes, bar + 1);
        bulk_g2s(smem + REG1 + HALF, To().w1lo, w1_bytes, bar + 1);
    };
    auto tma_online_w2 = [&] {
        mbar_expect_tx(bar + 2, 2 * w2_bytes);
        bulk_g2s(smem + REG3, To().w2, 2 * w2_bytes, bar + 2);
    };
    // AdamW streams W1 | b1 | W2 (one flat range; D % 4 == 0 keeps every 16-byte group inside one of the three) through the
    // ring: chunk k goes to slot k % ARING, whose barrier completes once per use
    const int an = d.ob2, nch = (an + ACH - 1) / ACH;
    auto aslot = [&](int s) { return smem + (s < 4 ? REG3 : REG1) + (s & 3) * ASLOT; };
    auto adam_issue = [&](int k) {
        const int off = k * ACH, s = k % ARING;
        const uint32_t bytes = 4u * (an - off < ACH ? an - off : ACH);
        char *dst = aslot(s);
        mbar_expect_tx(bar + 3 + s, 4 * bytes);
        bulk_g2s(dst, L.w + off, bytes, bar + 3 + s);
        bulk_g2s(dst + ACH * 4, L.m + off, bytes, bar + 3 + s);
        bulk_g2s(dst + ACH * 8, L.v + off, bytes, bar + 3 + s);
        bulk_g2s(dst + ACH * 12, L.vmax + off, bytes, bar + 3 + s);
    };
    // scheduled soft target update BEFORE round r's gradient step (deep_td_learning.py:283-284: (training_steps + 1) % freq == 0)
    auto soft_due = [&](int r) { return (L.steps0 + r + 2) % a.freq == 0; };
    // batch row tid of round r: its slot and the scalars of its record.  The slot is loaded first (row_slot), the record's
    // scalars (row_load) once it has arrived; row_store puts them where the round reads them.  The whole record is
    // prefetched into L2 for the round's row gathers.
    auto row_slot = [&](int r) { return L.slots[(size_t)r * a.B + tid]; };
    auto row_load = [&](int slot, uint32_t (&f)[3]) {
        const uint32_t *rec = L.records + (size_t)slot * W;
        for (int o = 0; o < W * 4; o += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char *>(rec) + o));
        f[0] = rec[a.lay.off_action]; f[1] = rec[a.lay.off_reward]; f[2] = rec[a.lay.off_flags];
    };
    auto row_store = [&](int slot, const uint32_t (&f)[3]) {
        mi.slot[tid] = slot;
        mi.act[tid] = (int)f[0];
        mi.rew[tid] = __uint_as_float(f[1]);
        mi.term[tid] = (f[2] & 1u) ? 1.f : 0.f;
        mi.cnt[tid] = (int)((f[2] >> 8) & 0xffffu);
    };
    const umma::Tile W2_hi = umma::make_tile(smem + REG3, 64, 128), W2_lo = umma::make_tile(smem + REG3 + 16384, 64, 128);
    const umma::Tile W2T_hi = umma::make_tile(smem + REG3 + 32768, 64, 128), W2T_lo = umma::make_tile(smem + REG3 + 49152, 64, 128);

    for (int round = 0; round < a.rounds; round++) {
        TC_STAMP(0);
        // ---- the row scalars of the launch's first round; those of every later round were loaded under the last AdamW sweep
        if (round == 0 && tid < a.B) {
            uint32_t f[3];
            const int slot = row_slot(0);
            row_load(slot, f);
            row_store(slot, f);
        }
        TC_STAMP(15);
        const bool soft_upd = soft_due(round);
        if (soft_upd) {
            // SU parameters per thread and pass, all loaded before the first store: a store to wt may alias a later load of w
            // for all the compiler knows, so one parameter at a time waited for an L2 round trip each.  The loads clamp their
            // index instead of branching (a branch here made ptxas serialise the kernel's wgmma, C7520).
            constexpr int SU = 16;
            for (int i0 = tid; i0 < d.P; i0 += SU * NTH) {
                float wv[SU], tv[SU];
#pragma unroll
                for (int u = 0; u < SU; u++) {
                    const int i = min(i0 + u * NTH, d.P - 1);
                    wv[u] = __ldcg(L.w + i); tv[u] = __ldcg(L.wt + i);
                }
#pragma unroll
                for (int u = 0; u < SU; u++)
                    if (i0 + u * NTH < d.P) L.wt[i0 + u * NTH] = soft_update(wv[u], tv[u], a.tau, a.omtau);
            }
            // The operand-layout tiles get the same elementwise update IN TILE ORDER (the hi tiles hold exactly the fp32 values of
            // the flat vectors, permuted; lo = residual of the new value): coalesced 16-byte accesses instead of rebuilding the
            // target tiles from the flat vector with scattered 4-byte stores.  Same function of the same inputs: bit-identical.
            // Four 16-byte groups per thread and pass, loaded before they are stored, as above.
            auto update_tile = [&](const float *on_hi, float *tg_hi, float *tg_lo, int n) {
                for (int i0 = tid * 4; i0 < n; i0 += 4 * NTH * 4) {
                    float4 w[4], t[4];
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        const int i = min(i0 + u * NTH * 4, n - 4);
                        w[u] = __ldcg(reinterpret_cast<const float4 *>(on_hi + i)); t[u] = __ldcg(reinterpret_cast<const float4 *>(tg_hi + i));
                    }
#pragma unroll
                    for (int u = 0; u < 4; u++) {
                        const int i = i0 + u * NTH * 4;
                        const float4 r = make_float4(soft_update(w[u].x, t[u].x, a.tau, a.omtau), soft_update(w[u].y, t[u].y, a.tau, a.omtau),
                                                     soft_update(w[u].z, t[u].z, a.tau, a.omtau), soft_update(w[u].w, t[u].w, a.tau, a.omtau));
                        if (i < n) {
                            *reinterpret_cast<float4 *>(tg_hi + i) = r;
                            *reinterpret_cast<float4 *>(tg_lo + i) = make_float4(tf32_lo(r.x), tf32_lo(r.y), tf32_lo(r.z), tf32_lo(r.w));
                        }
                    }
                }
            };
            update_tile(To().w1hi, Tt().w1hi, Tt().w1lo, HID * k1);
            update_tile(To().w2, Tt().w2, Tt().w2 + HID * HID, HID * HID);
            fence_proxy_async_all();
        }
        __syncthreads();

        // ================= phase T: y = max_a' Q_target(s', a') * gamma * (1 - term) + r =================
        TC_STAMP(1);
        // the target tiles (regions 1 and 3 are free: every product of the last round was waited for), unless the last round
        // issued them already: it does when no soft update falls on this round
        if (tid == 0 && (round == 0 || soft_upd)) tma_target();
        l1_issue(a, L, mi, smem, a.lay.off_next_state, h * 64, 0);
        if (soft_upd || round == 0) load_smalls(L.wt, d, mi.sm[1]);   // the target's small vectors only change at a soft update
        load_smalls(L.w, d, mi.sm[0]);   // the online ones are first read in phase O: they load under the wait for the target tiles
        umma::mbar_wait(bar + 0, round & 1);
        __syncthreads();
        TC_STAMP(2);
        for (int i = 0; i < ntiles; i++) {
            const int row0 = i * 128 + h * 64;
            float t1[32];
            layer1_block(a, L, mi, smem, a.lay.off_next_state, row0, t1);
            // chunk 0 of the next layer-1 block (the next row tile, or phase O's first) loads during the action loop
            if (i + 1 < ntiles) l1_issue(a, L, mi, smem, a.lay.off_next_state, row0 + 128, 0);
            else l1_issue(a, L, mi, smem, a.lay.off_state, h * 64, 0);
            const int rows[2] = {row0 + acc_row_here(0), row0 + acc_row_here(1)};
            int cnt[2];
            const uint8_t *ids[2];
            float best[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int p = 0; p < 2; p++) {
                cnt[p] = mi.cnt[rows[p]];
                ids[p] = (L.buf_flags & PRL_BUF_DYNAMIC_ACTIONS) ? reinterpret_cast<const uint8_t *>(L.records + (size_t)mi.slot[rows[p]] * W + a.lay.off_avail)
                                                                : kIota;
            }
            for (int act = 0; act < d.A; act++) {
                const int t4 = tid_here() & 3;
                float hi[32], lo[32], acc[32];
#pragma unroll
                for (int p = 0; p < 2; p++) {
                    // a select, not a branch: a conditional load here made ptxas serialise the kernel's wgmma (C7520)
                    const int id_l = ids[p][act], id = act < cnt[p] ? id_l : act;
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const float2 wv = lds2(&mi.sm[1].watb[id][8 * j + 2 * t4]);
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
                    const float2 w3v = lds2(&mi.sm[1].w3[8 * j + 2 * t4]);
                    const float2 b2v = lds2(&mi.sm[1].b2[8 * j + 2 * t4]);
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
        if (tid == 0) { tma_online_w1(); tma_online_w2(); }
        TC_STAMP(4);
        // weight-gradient accumulators; both warpgroups issue the same products on different output columns:
        // gw2 = dW2 columns [32 h, 32 h + 32), gb2 = [db2 | .] (column 0 of dZ2^T E, the same on both warpgroups),
        // gw1 = dW1s columns [NW h, NW h + NW), for NW = 64 its transpose: dW1s^T rows [64 h, 64 h + 64),
        // gba = [db1 | dW1a] columns [16 h, 16 h + 16) (0 = bias, 1 + k = action k)
        float gw2[16], gb2[4], gw1[NW / 2], gba[8];
        float mae_acc = 0.f, db3_acc = 0.f;
        float *arena = reinterpret_cast<float *>(smem);
        const umma::Tile TA_hi = umma::make_tile(smem + AR_A_HI, 64, TL), TA_lo = umma::make_tile(smem + AR_A_LO, 64, TL);
        const umma::Tile TB_hi = umma::make_tile(smem + AR_B_HI, 64, TL), TB_lo = umma::make_tile(smem + AR_B_LO, 64, TL);
        const umma::Tile TE = umma::make_tile(smem + AR_E, 64, TL);
        // E^T = [1 | onehot(action)]^T of the 64 rows from row b0 (this thread: columns rA, rB of the tile, rows 8 t4 .. + 8)
        auto e_scatter = [&](int b0, int rA, int rB, int t4) {
#pragma unroll
            for (int p = 0; p < 2; p++) {
                const int r = p ? rB : rA, act = mi.act[b0 + r];
#pragma unroll
                for (int x = 0; x < 8; x++) {
                    const int er = t4 * 8 + x;
                    arena[AR_E / 4 + umma::tile_index2(er, r, 64, TL)] = (er == 0 || er == act + 1) ? 1.f : 0.f;
                }
            }
        };
        for (int i = 0; i < ntiles; i++) {
            const int row0 = i * 128 + h * 64;
            if (i > 0) {   // the last tile's passes overwrote regions 1 and 3 (tile 0's first chunk was issued in phase T)
                if (tid == 0) { tma_online_w1(); tma_online_w2(); }
                l1_issue(a, L, mi, smem, a.lay.off_state, row0, 0);
            }
            // bar[1] and bar[2] complete once per row tile (a parity computed here, not carried across the chains)
            umma::mbar_wait(bar + 1, (uint32_t)(round * ntiles + i) & 1u);
            __syncthreads();
            const int rows[2] = {row0 + acc_row_here(0), row0 + acc_row_here(1)};
            float h1[32], z[32], hi[32], lo[32];
            layer1_block(a, L, mi, smem, a.lay.off_state, row0, h1);
            __syncthreads();   // both warpgroups are done with the W1 tiles: region 1 takes H1 and dZ2 below
            if (i == 0) TC_STAMP(5);
            int ai[2];
#pragma unroll
            for (int p = 0; p < 2; p++) {
                ai[p] = mi.act[rows[p]];
#pragma unroll
                for (int j = 0; j < 8; j++) {
                    const float2 wv = lds2(&mi.sm[0].watb[ai[p]][8 * j + 2 * t4]);
                    h1[4 * j + 2 * p] = fmaxf(h1[4 * j + 2 * p] + wv.x, 0.f);
                    h1[4 * j + 2 * p + 1] = fmaxf(h1[4 * j + 2 * p + 1] + wv.y, 0.f);
                }
            }
            // H1 and dZ2 wait in this warpgroup's half of region 1 (the W1 tiles are dead) while dZ2 and dH1 are formed:
            // values that stay live across a wgmma chain besides its own operands cost the registers the chain needs, and
            // ptxas serialises every wgmma of the kernel when a chain does not fit (C7511).  The staging buffers in region 2
            // keep this tile's state rows for dW1s.
            float *h1s = reinterpret_cast<float *>(smem + REG1 + h * HALF) + (tid & 127);
#pragma unroll
            for (int c = 0; c < 32; c++) h1s[c * 128] = h1[c];
            umma::mbar_wait(bar + 2, (uint32_t)(round * ntiles + i) & 1u);   // W2 | W2^T, loaded under layer 1
            acc_to_frag(h1, hi, lo);
            umma::gemm3_rs<HID, 8>(z, hi, lo, W2_hi, W2_lo, false);
            umma::wg_commit();
            umma::wg_wait<0>();
            float part[2] = {0.f, 0.f}, dq[2];
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const float2 w3v = lds2(&mi.sm[0].w3[8 * j + 2 * t4]);
                const float2 b2v = lds2(&mi.sm[0].b2[8 * j + 2 * t4]);
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
                const float2 w3v = lds2(&mi.sm[0].w3[8 * j + 2 * t4]);
                mi.dw3[2 * j][tid] = (i == 0 ? 0.f : mi.dw3[2 * j][tid]) + (dq[0] * z[4 * j] + dq[1] * z[4 * j + 2]);
                mi.dw3[2 * j + 1][tid] = (i == 0 ? 0.f : mi.dw3[2 * j + 1][tid]) + (dq[0] * z[4 * j + 1] + dq[1] * z[4 * j + 3]);
#pragma unroll
                for (int p = 0; p < 2; p++) {
                    z[4 * j + 2 * p] = z[4 * j + 2 * p] > 0.f ? dq[p] * w3v.x : 0.f;
                    z[4 * j + 2 * p + 1] = z[4 * j + 2 * p + 1] > 0.f ? dq[p] * w3v.y : 0.f;
                }
            }
            float dz1[32];
#pragma unroll
            for (int c = 0; c < 32; c++) h1s[(32 + c) * 128] = z[c];   // dZ2 waits there too
            acc_to_frag(z, hi, lo);
            umma::gemm3_rs<HID, 8>(dz1, hi, lo, W2T_hi, W2T_lo, false);   // dH1 = dZ2 W2
            umma::wg_commit();
            umma::wg_wait<0>();
#pragma unroll
            for (int c = 0; c < 32; c++) {
                h1[c] = h1s[c * 128];
                z[c] = h1s[(32 + c) * 128];
                dz1[c] = (h1[c] > 0.f) ? dz1[c] : 0.f;
            }
            // dZ1 waits in region 3's W2 half until its dW1s pass, so that it is not live in registers across the other
            // passes' chains; written once both warpgroups are done with W2
            __syncthreads();
            float *dzs = reinterpret_cast<float *>(smem + REG3 + h * (HALF / 2)) + (tid & 127);
#pragma unroll
            for (int c = 0; c < 32; c++) dzs[c * 128] = dz1[c];
            if (i == 0) TC_STAMP(6);

            // ---- weight gradients: contractions over the batch rows, 64 rows (one warpgroup's block) per pass; the owner of the
            //      block scatters the transposes of its rows while the other warpgroup builds E^T.  The dW2 | db2 passes over
            //      both blocks come first, then the dW1s | [db1 | dW1a] passes: every output element still accumulates the
            //      blocks in the same order, and no H1 or dZ2 stays live across the register-fed dW1s chain.
            for (int hf = 0; hf < 2; hf++) {
                const int ft = tid_here(), h = ft >> 7, t4 = ft & 3, lane = ft & 31, warp = ft >> 5, rA = acc_row_here(0), rB = rA + 8;
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
                } else {
                    e_scatter(i * 128 + hf * 64, rA, rB, t4);
                }
                umma::fence_async_smem();
                __syncthreads();
                if (first) TC_STAMP(11);
                umma::gemm3<32>(gw2, TA_hi, TA_lo, TB_hi.rows_from(32 * h), TB_lo.rows_from(32 * h), 64, !first);
                umma::gemm3<8>(gb2, TA_hi, TA_lo, TE, TE, 64, !first, false, true);
                umma::wg_commit();
                if (NW < 64 && lane < 16 && 32 * (lane & 3) < d.obs) {   // the state rows of this block for S^T, into L1:
                    // lane 4 ri + c = 128-byte line c of row warp + 8 ri
                    const float *src = reinterpret_cast<const float *>(L.records + (size_t)mi.slot[i * 128 + hf * 64 + warp + 8 * (lane >> 2)] * W) +
                                       a.lay.off_state + 32 * (lane & 3);
                    asm volatile("prefetch.global.L1 [%0];" ::"l"(src));
                }
                umma::wg_wait<0>();
                if (first) TC_STAMP(12);
            }
            for (int hf = 0; hf < 2; hf++) {
                const int ft = tid_here(), h = ft >> 7, t4 = ft & 3, lane = ft & 31, warp = ft >> 5, rA = acc_row_here(0), rB = rA + 8;
                const bool mine = h == hf;
                const bool first = (i == 0 && hf == 0);
                __syncthreads();   // previous products have been waited for: the arena is free
                // NW < 64 (obs <= 64): S^T is built as a B tile.  Every warp reads whole state rows of this half coalesced
                // (lane = k) and scatters them into column rq of the transposed tile.
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
                if constexpr (NW < 64) st_rows_load(0);
                if (mine) {
#pragma unroll
                    for (int j = 0; j < 8; j++)
#pragma unroll
                        for (int p = 0; p < 2; p++)
#pragma unroll
                            for (int e = 0; e < 2; e++) {
                                const int idx = umma::tile_index2(8 * j + 2 * t4 + e, p ? rB : rA, 64, TL), c = 4 * j + 2 * p + e;
                                const float v = reinterpret_cast<const float *>(smem + REG3 + h * (HALF / 2))[c * 128 + (ft & 127)];
                                arena[AR_A_HI / 4 + idx] = v; arena[AR_A_LO / 4 + idx] = tf32_lo(v);               // dZ1^T
                            }
                } else {
                    e_scatter(i * 128 + hf * 64, rA, rB, t4);
                }
                if constexpr (NW < 64) {
                    st_rows_scatter(0);
                    st_rows_load(4);
                    st_rows_scatter(4);
                }
                umma::fence_async_smem();
                __syncthreads();
                if (first) TC_STAMP(13);
                if constexpr (NW == 64) {
                    // dW1s^T = S^T dZ1 (obs rows [64 h, 64 h + 64) on warpgroup h): A = S^T as register fragments read from the
                    // owner's layer-1 staging buffer of K chunk h, B = the dZ1^T tile.  Each element gets the same three
                    // products over the same K steps as dZ1^T S, the small terms in the same order (B_LO_FIRST).
                    const float *sbuf = reinterpret_cast<const float *>(smem + REG2 + hf * 2 * SBUF + h * SBUF);
                    float shi[32], slo[32];
#pragma unroll
                    for (int ks = 0; ks < 8; ks++)
#pragma unroll
                        for (int q = 0; q < 2; q++)
#pragma unroll
                            for (int p = 0; p < 2; p++) {
                                const int o = p ? rB : rA, r = 8 * ks + t4 + 4 * q;   // A row = obs column, K = batch row
                                umma::split_tf32(sbuf[r * 64 + (((o >> 2) ^ (r & 7)) << 2) + (o & 3)], shi[4 * ks + 2 * q + p], slo[4 * ks + 2 * q + p]);
                            }
                    umma::gemm3_rs<64, 8, true>(gw1, shi, slo, TA_hi, TA_lo, !first);
                } else {
                    umma::gemm3<NW>(gw1, TA_hi, TA_lo, TB_hi.rows_from(NW * h), TB_lo.rows_from(NW * h), 64, !first);
                }
                umma::gemm3<16>(gba, TA_hi, TA_lo, TE.rows_from(16 * h), TE.rows_from(16 * h), 64, !first, false, true);
                umma::wg_commit();
                umma::wg_wait<0>();
                if (first) TC_STAMP(14);
            }
            umma::fence_async_smem();   // the arena was written through the generic proxy, the next W1 copy is a TMA write
            __syncthreads();            // the arena is free: the next tile's W1 copy / the gradient staging may overwrite it
        }
        // regions 3 (W2 / W2^T; the arena's TB hi tile, fenced above) and 1 (the rest of the arena) are free: AdamW's
        // first chunks load during the gradient staging.
        // Issuing them under the last tile's weight-gradient products instead made the kernel slower.
        if (a.adam_tma && tid == 0)
            for (int k = 0; k < ARING && k < nch; k++) adam_issue(k);
        // this round's row scalars are dead: the next round's are loaded under AdamW and stored at its end.  Its target tiles
        // are issued after the sweep unless a soft update, which rewrites them, comes first.
        const bool next_rows = round + 1 < a.rounds && tid < a.B;
        const bool stage_target = round + 1 < a.rounds && !soft_due(round + 1);
        int nslot = 0;
        uint32_t nf[3];
        if (next_rows) nslot = row_slot(round + 1);

        TC_STAMP(8);
        // ================= AdamW ==========
        // column sums of dW3 over the warp's rows: lanes with equal lane % 4 hold the same columns
#pragma unroll
        for (int c = 0; c < 16; c++) {
            float v = mi.dw3[c][tid];
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
                const int j = acc_row_here(p);                         // the gradient's row = hidden unit
#pragma unroll
                for (int jb = 0; jb < 4; jb++)
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const int c = 8 * jb + 2 * t4 + e, x = 4 * jb + 2 * p + e;
                        gs_w2[j * 65 + 32 * h + c] = gw2[x];
                        if (NW < 64 && jb < NW / 8 && NW * h + c < d.obs) gs_w1[j * pitch1 + NW * h + c] = gw1[x];
                        if (jb < 2) {
                            const int ce = 16 * h + c;
                            if (ce == 0) gs_b1[j] = gba[x];
                            else if (ce - 1 < d.A) gs_w1[j * pitch1 + d.obs + ce - 1] = gba[x];
                        }
                    }
                if constexpr (NW == 64) {   // gw1 holds dW1s^T: this thread's row p is obs column 64 h + j
                    const int k = 64 * h + j;
#pragma unroll
                    for (int jb = 0; jb < 8; jb++)
#pragma unroll
                        for (int e = 0; e < 2; e++)
                            if (k < d.obs) gs_w1[(8 * jb + 2 * t4 + e) * pitch1 + k] = gw1[4 * jb + 2 * p + e];
                }
                if (h == 0 && t4 == 0) gs_b2[j] = gb2[2 * p];
            }
            __syncthreads();
            TC_STAMP(7);
            if (next_rows) row_load(nslot, nf);
            // 2) AdamW over the flat parameter vector, all 256 threads.  The sweep is bound by L2 round trips, not bytes: W1 | b1 |
            //    W2 arrive by TMA in chunks of ACH parameters through an ARING-slot ring in regions 3 and 1, up to 128 KB of
            //    loads in flight and no thread holding load registers.  The loads of the small vectors (b1 | b2 | W3 | b3,
            //    one parameter per thread) are in flight across the whole sweep.
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
            if (a.adam_tma) {
                // one 16-byte group of chunk k per thread: w | m | v | vmax from the chunk's ring slot (TMA), the gradient from
                // the staging, the results to global memory with 16-byte stores; b1's groups ride along and are left to the tail
                const int n1 = HID * d.D;
                for (int k = 0; k < nch; k++) {
                    const int s = k % ARING, uses = (nch - 1 - s) / ARING + 1;
                    umma::mbar_wait(bar + 3 + s, (uint32_t)(round * uses + k / ARING) & 1u);
                    const int i = k * ACH + 4 * tid;
                    if (i < an && (i < n1 || i >= d.oW2)) {
                        const float4 *sl = reinterpret_cast<const float4 *>(aslot(s)) + tid;
                        float4 w = sl[0], mm = sl[ACH / 4], vv = sl[ACH / 2], xx = sl[3 * ACH / 4];
                        float *gp;
                        if (i < n1) {
                            const int row = i / d.D, c = i - row * d.D;
                            gp = gs_w1 + row * pitch1 + c;
                        } else {
                            const int e = i - d.oW2;
                            gp = gs_w2 + (e >> 6) * 65 + (e & 63);
                        }
                        w.x = adam_math(w.x, mm.x, vv.x, xx.x, gp[0], hs); w.y = adam_math(w.y, mm.y, vv.y, xx.y, gp[1], hs);
                        w.z = adam_math(w.z, mm.z, vv.z, xx.z, gp[2], hs); w.w = adam_math(w.w, mm.w, vv.w, xx.w, gp[3], hs);
                        *reinterpret_cast<float4 *>(L.w + i) = w; *reinterpret_cast<float4 *>(L.m + i) = mm;
                        *reinterpret_cast<float4 *>(L.v + i) = vv; *reinterpret_cast<float4 *>(L.vmax + i) = xx;
                        // the new value replaces its gradient in the staging: the operand tiles are built from there below
                        gp[0] = w.x; gp[1] = w.y; gp[2] = w.z; gp[3] = w.w;
                    }
                    if (k + ARING < nch) {   // every thread is done with slot s: refill it with chunk k + ARING
                        __syncthreads();
                        if (tid == 0) adam_issue(k + ARING);
                    }
                }
                __syncthreads();
                // the ring is consumed and regions 1 and 3 are free: the next round's target tiles load under the tile pass
                if (tid == 0 && stage_target) tma_target();
                // The operand-layout tiles from the new W1 | W2 in the staging, one 16-byte group of a tile per thread and
                // store, in tile order: coalesced, where the sweep's own order scattered them (16-byte pieces of W1 and W2
                // into separate sectors, W2^T one float at a time), which made the tile stores most of the sweep's store
                // traffic.  A group is row r, columns k .. k + 3 of the tile (umma::tile_index).
                auto group_rc = [](int p, int K, int &r, int &k) {
                    const int rem = p % (8 * K);
                    r = p / (8 * K) * 8 + ((rem >> 2) & 7);
                    k = (rem >> 5) * 4;
                };
                auto put = [](float *hi, float *lo, int p, float4 x) {
                    *reinterpret_cast<float4 *>(hi + p) = x;
                    *reinterpret_cast<float4 *>(lo + p) = make_float4(tf32_lo(x.x), tf32_lo(x.y), tf32_lo(x.z), tf32_lo(x.w));
                };
                // kperm^-1: the W2 column at K position t of a kperm-ordered tile
                auto kinv = [](int t) { return (t & ~7) | ((t & 3) << 1) | ((t >> 2) & 1); };
                const NetTiles t = To();
                for (int p = 4 * tid; p < HID * k1; p += 4 * NTH) {   // W1: columns from obs on stay zero
                    int r, k;
                    group_rc(p, k1, r, k);
                    if (k < d.obs) {
                        const float *g = gs_w1 + r * pitch1 + k;
                        put(t.w1hi, t.w1lo, p, make_float4(g[0], g[1], g[2], g[3]));
                    }
                }
                for (int p = 4 * tid; p < HID * HID; p += 4 * NTH) {
                    int r, k;
                    group_rc(p, HID, r, k);
                    const float *g = gs_w2 + r * 65;   // W2 tile: row r, K positions k .. k + 3 = columns kinv(k + q)
                    put(t.w2, t.w2 + 4096, p, make_float4(g[kinv(k)], g[kinv(k + 1)], g[kinv(k + 2)], g[kinv(k + 3)]));
                    // W2^T tile: row r = W2 column, K positions k .. k + 3 = W2 rows kinv(k + q)
                    put(t.w2t, t.w2t + 4096, p, make_float4(gs_w2[kinv(k) * 65 + r], gs_w2[kinv(k + 1) * 65 + r],
                                                            gs_w2[kinv(k + 2) * 65 + r], gs_w2[kinv(k + 3) * 65 + r]));
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
                if (tid == 0 && stage_target) tma_target();
                rebuild_tiles(L.w, d, To(), tid);         // D % 4 != 0 or unaligned parameters: tiles from the flat vector
            }
            TC_STAMP(10);
            fence_proxy_async_all();                    // the tile writes and W1 | W2 are read by TMA in the next round
            if (si >= 0) {
                L.w[si] = adam_math(sw, sm, sv2, sx, sg, hs);
                L.m[si] = sm; L.v[si] = sv2; L.vmax[si] = sx;
            }
        }
        if (next_rows) row_store(nslot, nf);
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
    // AdamW streams the flat parameters and moments by TMA bulk copies (16-byte granules): every group of 4 parameters
    // must stay inside one of W1 / b1 / W2 and every pointer must be 16-byte aligned, else the scalar sweep runs
    bool adam_tma = ((c.obs_dim + c.n_actions) & 3) == 0;
    for (int i = 0; i < count; i++) {
        prl_dqn *q = dqns[i];
        prl_buf *b = bufs[i];
        PRL_REQUIRE(q && b, "null learner / buffer");
        // a shard's sampler draws global slots in [0, capacity * world); the learner indexes its local records with them
        PRL_REQUIRE(b->shard_world <= 1, "buffer %d is one shard of a multi-GPU buffer: the tensor-core learner samples local buffers only", i);
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
        adam_tma = adam_tma && (((uintptr_t)q->w | (uintptr_t)q->m | (uintptr_t)q->v | (uintptr_t)q->vmax) & 15) == 0;
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
    a.adam_tma = adam_tma ? 1 : 0;
    a.prof = q0->prof;
    { static const int c = [] { const char *e = getenv("PRL_TC_PROF_CTA"); return e ? atoi(e) : 0; }(); a.prof_cta = c; }
    const size_t smem = MISC_OFF + sizeof(Misc);
    PRL_REQUIRE(smem <= (size_t)q0->max_smem, "tensor-core learner needs %zu B of shared memory", smem);
    const int nw = dw1_share(c.obs_dim);
    void (*const kern)(TcArgs) = nw == 64 ? k_dqn_tc<64> : nw == 32 ? k_dqn_tc<32> : nw == 16 ? k_dqn_tc<16> : k_dqn_tc<8>;
    PRL_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));

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
        kern<<<count, NTH, smem, stream>>>(a);
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
