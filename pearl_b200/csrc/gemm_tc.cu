// gemm_tc.cu — the actor-critic learners' contraction (gemm.cuh: C[i][j] = sum_c A(i, c) * B(j, c)) on Hopper's tensor
// cores: wgmma.mma_async of kind tf32 with the 3xTF32 operand split of umma.cuh (hi*hi + hi*lo + lo*hi accumulated in
// fp32 registers), so the products keep fp32 parity with the reference's torch matmuls (1e-4 gate).
//
// One CTA (two warpgroups) computes a 128 x TN tile of C (TN = 64 or 32), each warpgroup 64 rows of it.  The contraction
// axis is walked in chunks of 32:
//   * all 8 warps read the chunk's A (128 x 32) and B (TN x 32) elements from global memory exactly as gemm.cuh's `Mat`
//     describes them (two concatenated sources, a ones column, stacked networks; either the row or the feature axis of
//     the Mat is the contraction axis), TWO chunks ahead of the one being multiplied (three register sets), split them
//     into hi / lo and store them as 16-byte chunks into K-major no-swizzle tiles with a 144-byte chunk pitch — with that
//     pitch both global layouts give conflict-free STS.128 and fully coalesced global loads;
//   * three shared-memory stages, the products of one chunk stay in flight while the next chunk is stored;
//   * epilogue: the register accumulators are staged through shared memory so that bias / mask / accumulate reads and
//     the C stores are coalesced along j.
// gemm_tc_launch sends products with fewer than 4096 output rows to the SIMT tiles.  That threshold was chosen for the
// tcgen05 kernel this one replaces and has not been measured again on H100 (tools/gemm_bench.py times both engines).
#include "gemm.cuh"
#include "umma.cuh"

namespace prl {

int g_contraction_engine = 1;   // 1: tensor-core tiles, 0: SIMT tiles (prl_set_contraction_engine)

namespace {

constexpr int TM = 128, GKT = 32, LBO = 144, SBO = 8 * LBO, NSTAGE = 3, NSET = 3, NLOAD = 256;

// which (row of the tile, 16-byte K chunk) a thread's slot u covers.  XO: the Mat's rows are the tile's rows (features are
// contracted, contiguous along k): 8 lanes read one row's 128 contiguous bytes.  !XO: the Mat's rows are contracted
// (contiguous along the tile's row index): 32 lanes read 32 consecutive tile rows of one Mat row.
template <int ROWS, bool XO>
__device__ __forceinline__ void slot_coords(int u, int w, int lane, int &r, int &kc) {
    if (XO) {
        r = w * (ROWS / 8) + u * 4 + (lane >> 3);
        kc = lane & 7;
    } else {
        constexpr int NRB = ROWS / 32;
        r = (w % NRB) * 32 + lane;
        kc = (w / NRB) * NRB + u;
    }
}

// One operand (ROWS x 32 per chunk) as seen by one loader thread.  Everything that does not change from chunk to chunk
// is computed once.  Loads never need a predicate: indices are clamped into the operand (a tile row past the operand's
// extent repeats its last row — its products land in rows / columns of C that the epilogue never stores — and an index past
// the end of the contraction axis repeats the last one and is zeroed when the tile is stored).  The loop body is kept
// small on purpose: the first version inlined four paths per operand and ran out of the instruction cache at ~10 clocks
// per instruction.
template <int ROWS, bool XO>
struct Operand {
    static constexpr int S = ROWS / 32;
    const Mat &m;
    int Kc, kc4;                // contraction length; XO: this thread's 16-byte chunk (floats) inside a 32-deep chunk
    const float *zb1, *zb2;     // part bases with the network offset applied (zb2 also with -split)
    int off1[S], off2[S];       // XO: float offset of the slot's row in part 1 / part 2
    int kcu[S];                 // !XO: first contraction index of slot u inside a chunk
    int soff[S];                // byte offset of the slot's 16-byte chunk inside the operand tile
    const float *fbase;         // !XO: this thread's feature column
    int fld;                    // !XO: its row pitch
    bool isone, vec1, vec2;

    __device__ __forceinline__ Operand(const Mat &m_, int z, int out0, int out_lim, int Kc_, int w, int lane) : m(m_), Kc(Kc_) {
        zb1 = m.p1 + z * m.net_stride1;
        zb2 = m.p2 + z * m.net_stride2 - m.split;
        fbase = zb1; fld = 0; isone = false; kc4 = 0; vec1 = vec2 = false;
#pragma unroll
        for (int u = 0; u < S; u++) {
            int r, kc;
            slot_coords<ROWS, XO>(u, w, lane, r, kc);
            soff[u] = (r >> 3) * SBO + kc * LBO + (r & 7) * 16;
            kcu[u] = kc * 4;
            const int row = min(out0 + r, out_lim - 1);
            off1[u] = XO ? row * m.ld1 : 0;
            off2[u] = XO ? row * m.ld2 : 0;
            if (XO) kc4 = kc * 4;
        }
        if (XO) {
            vec1 = ((reinterpret_cast<uintptr_t>(zb1) & 15) | (m.ld1 & 3)) == 0;
            vec2 = m.p2 != nullptr && ((reinterpret_cast<uintptr_t>(zb2) & 15) | (m.ld2 & 3)) == 0;
        } else {
            int r, kc;
            slot_coords<ROWS, XO>(0, w, lane, r, kc);
            const int out = out0 + r;
            isone = out == m.ones_at && out < out_lim;
            int f = min(out, out_lim - 1);
            if (f == m.ones_at) f = 0;                      // any valid address: the value is replaced by 1.0 / never used
            fbase = f < m.split ? zb1 + f : zb2 + f;
            fld = f < m.split ? m.ld1 : m.ld2;
        }
    }
    // XO: chunk c lies inside one source, away from the end of the contraction axis and the ones column
    __device__ __forceinline__ bool interior(int f0) const {
        return f0 + GKT <= Kc && (f0 + GKT <= m.split || f0 >= m.split) && !(m.ones_at >= f0 && m.ones_at < f0 + GKT);
    }
    __device__ __forceinline__ void fetch(int c, float (&reg)[S][4]) const {
        const int f0 = c * GKT;
        if (XO) {
            const bool second = f0 >= m.split;
            if (interior(f0) && (second ? vec2 : vec1)) {
                const float *base = (second ? zb2 : zb1) + f0 + kc4;
#pragma unroll
                for (int u = 0; u < S; u++) {
                    const float4 q = __ldg(reinterpret_cast<const float4 *>(base + (second ? off2[u] : off1[u])));
                    reg[u][0] = q.x; reg[u][1] = q.y; reg[u][2] = q.z; reg[u][3] = q.w;
                }
            } else {
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    int f = min(f0 + kc4 + e, Kc - 1);
                    if (f == m.ones_at) f = 0;
                    const bool sec = f >= m.split;
                    const float *base = (sec ? zb2 : zb1) + f;
#pragma unroll
                    for (int u = 0; u < S; u++) reg[u][e] = __ldg(base + (sec ? off2[u] : off1[u]));
                }
            }
        } else if (isone) {                      // the ones column (bias gradient): no load, the stored value is 1
#pragma unroll
            for (int u = 0; u < S; u++)
#pragma unroll
                for (int e = 0; e < 4; e++) reg[u][e] = 1.f;
        } else if (f0 + GKT <= Kc) {
#pragma unroll
            for (int u = 0; u < S; u++) {
                const float *q = fbase + (size_t)(f0 + kcu[u]) * fld;
#pragma unroll
                for (int e = 0; e < 4; e++) reg[u][e] = __ldg(q + (size_t)e * fld);
            }
        } else {
#pragma unroll
            for (int u = 0; u < S; u++)
#pragma unroll
                for (int e = 0; e < 4; e++) reg[u][e] = __ldg(fbase + (size_t)min(f0 + kcu[u] + e, Kc - 1) * fld);
        }
    }
    __device__ __forceinline__ bool edge(int c) const { return XO ? !interior(c * GKT) : c * GKT + GKT > Kc; }
    // the value of element (slot u, e) of an EDGE chunk as the product sees it (ones column, zero past the contraction axis);
    // in every other chunk it is the loaded value itself
    __device__ __forceinline__ float edge_elem(int c, int u, int e, float loaded) const {
        const int con = c * GKT + (XO ? kc4 : kcu[u]) + e;
        float v = loaded;
        if (XO && con == m.ones_at) v = 1.f;
        if (con >= Kc) v = 0.f;
        return v;
    }
    // split into hi (the value itself: the tensor core truncates) / lo and store as 16-byte chunks of the operand tiles
    __device__ __forceinline__ void store(int c, const float (&reg)[S][4], unsigned char *hi, unsigned char *lo) const {
        if (edge(c)) {                               // uniform branch, taken for at most two chunks of a product
#pragma unroll
            for (int u = 0; u < S; u++) {
                float v[4], l[4];
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    v[e] = edge_elem(c, u, e, reg[u][e]);
                    l[e] = v[e] - __uint_as_float(__float_as_uint(v[e]) & 0xffffe000u);
                }
                *reinterpret_cast<float4 *>(hi + soff[u]) = make_float4(v[0], v[1], v[2], v[3]);
                *reinterpret_cast<float4 *>(lo + soff[u]) = make_float4(l[0], l[1], l[2], l[3]);
            }
            return;
        }
#pragma unroll
        for (int u = 0; u < S; u++) {
            float l[4];
#pragma unroll
            for (int e = 0; e < 4; e++) l[e] = reg[u][e] - __uint_as_float(__float_as_uint(reg[u][e]) & 0xffffe000u);
            *reinterpret_cast<float4 *>(hi + soff[u]) = make_float4(reg[u][0], reg[u][1], reg[u][2], reg[u][3]);
            *reinterpret_cast<float4 *>(lo + soff[u]) = make_float4(l[0], l[1], l[2], l[3]);
        }
    }
};

// Both warpgroups' accumulators (rows 64 wg .. of the tile) -> C, staged through shared memory (the operand stages are
// free: every product has completed) so that the bias / mask / accumulate reads and the C stores are coalesced along C's
// contiguous axis.  SWAP: the accumulator is C transposed (tile rows = C's column index).
template <int TN, bool SWAP>
__device__ __forceinline__ void epilogue(const GemmArgs &g, int z, const float *d, float *tb, int a0, int b0) {
    const int tid = threadIdx.x, wg = tid >> 7;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < TN / 8; j++)
#pragma unroll
        for (int p = 0; p < 2; p++)
#pragma unroll
            for (int e = 0; e < 2; e++) tb[(wg * 64 + umma::acc_row(p)) * (TN + 1) + umma::acc_col(j, e)] = d[4 * j + 2 * p + e];
    __syncthreads();
    for (int o = tid; o < TM * TN; o += NLOAD) {
        const int r = SWAP ? o % TM : o / TN, c = SWAP ? o / TM : o % TN;
        const int i = SWAP ? b0 + c : a0 + r, j = SWAP ? a0 + r : b0 + c;
        if (i < (SWAP ? g.No : g.Mo) && j < (SWAP ? g.Mo : g.No)) gemm_emit(g, z, i, j, tb[r * (TN + 1) + c]);
    }
}

// SS form: 8 warps = two warpgroups; every thread is loader and consumer.  Per chunk: store the chunk's tiles into stage
// c % 3, make them visible to the tensor core, one block barrier, then each warpgroup issues the 12 wgmma of its 64 rows
// (4 K-steps x 3 split terms) and leaves them in flight: the wait before the NEXT barrier only asks for the chunk before
// to have completed, which is what frees the stage written after that barrier.
template <int TN, bool AO, bool BO>
__global__ void __launch_bounds__(NLOAD, 1) k_gemm_tc(const GemmArgs g) {
    extern __shared__ __align__(128) unsigned char dsm[];
    constexpr int A_B = (TM / 8) * SBO, B_B = (TN / 8) * SBO, STAGE_B = 2 * A_B + 2 * B_B;
    const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31, wg = tid >> 7, z = blockIdx.z;
    const int i0 = blockIdx.x * TM, j0 = blockIdx.y * TN;
    const int nch = (g.Kc + GKT - 1) / GKT;
    const uint32_t base = umma::smem_u32(dsm);

    const Operand<TM, AO> opA(g.A, z, i0, g.Mo, g.Kc, w, lane);
    const Operand<TN, BO> opB(g.B, z, j0, g.No, g.Kc, w, lane);
    float ra[NSET][TM / 32][4], rb[NSET][TN / 32][4];
    float d[TN / 2];
#pragma unroll
    for (int p = 0; p < NSET - 1; p++)
        if (p < nch) { opA.fetch(p, ra[p]); opB.fetch(p, rb[p]); }
    static_assert(NSET == NSTAGE, "stage index == register set index");
    for (int c0 = 0; c0 < nch; c0 += NSET) {
#pragma unroll
        for (int u = 0; u < NSET; u++) {
            const int c = c0 + u;
            if (c < nch) {
                if (c + NSET - 1 < nch) {       // two chunks ahead of the one being stored
                    opA.fetch(c + NSET - 1, ra[(u + NSET - 1) % NSET]);
                    opB.fetch(c + NSET - 1, rb[(u + NSET - 1) % NSET]);
                }
                unsigned char *st = dsm + u * STAGE_B;
                opA.store(c, ra[u], st, st + A_B);
                opB.store(c, rb[u], st + 2 * A_B, st + 2 * A_B + B_B);
                umma::fence_async_smem();       // generic-proxy writes -> visible to the tensor core's async proxy
                umma::wg_wait<1>();             // chunk c - 2 has completed: after the barrier its stage may be overwritten
                __syncthreads();
                const umma::Tile ah{base + u * STAGE_B + wg * (64 / 8) * SBO, LBO, SBO}, al = ah.shifted(A_B);
                const umma::Tile bh{base + u * STAGE_B + 2 * A_B, LBO, SBO}, bl = bh.shifted(B_B);
                umma::gemm3<TN>(d, ah, al, bh, bl, GKT, c > 0);
                umma::wg_commit();
            }
        }
    }
    umma::wg_wait<0>();
    epilogue<TN, false>(g, z, d, reinterpret_cast<float *>(dsm), i0, j0);
}

// ---- RS form: the A operand lives in registers ---------------------------------------------------------------------
// The SS kernel above moves 120 KB through shared memory per 32-deep chunk of a 128 x 64 tile (48 KB of hi / lo stores and
// 72 KB of operand reads by the 12 MMAs).  Here the 128-row operand never touches shared memory: it must be the operand
// whose Mat has the tile rows along the contiguous axis ("rows contracted"); every thread loads exactly the elements of
// its own wgmma A fragments (8 consecutive tile rows x 4 contraction indices per warp and load: whole 32-byte sectors).
// Shared memory only carries the TN-row operand: 16 KB of stores + 24 KB of MMA reads per chunk.  The fragments of a chunk
// are the operands of products in flight, so a chunk's products are waited for before the next chunk's split.
//   nn.Linear forward     D[n][m] = sum_k Wt[k][n] x[m][k]     A = a transposed copy of W kept by the learner, SWAP
//   backward-data         D[k][m] = sum_n W[n][k] dy[m][n]      A = W as stored, SWAP
//   backward-weight       D[n][k] = sum_m dy[m][n] x[m][k]      A = dy as stored
// SWAP: the accumulator is C transposed (tile rows = C's column index).
struct FragA {
    const float *base[2];   // this thread's two tile rows (Mat features) at contraction index 0
    int fld[2];
    bool one[2];
    int Kc, t;
    __device__ __forceinline__ FragA(const Mat &m, int z, int out0, int out_lim, int Kc_) : Kc(Kc_), t(threadIdx.x & 3) {
        const float *zb1 = m.p1 + z * m.net_stride1, *zb2 = m.p2 + z * m.net_stride2 - m.split;
#pragma unroll
        for (int p = 0; p < 2; p++) {
            const int out = out0 + (threadIdx.x >> 7) * 64 + umma::acc_row(p);
            one[p] = out == m.ones_at && out < out_lim;
            int f = min(out, out_lim - 1);
            if (f == m.ones_at) f = 0;                      // any valid address: the value is replaced by 1.0 / never used
            base[p] = f < m.split ? zb1 + f : zb2 + f;
            fld[p] = f < m.split ? m.ld1 : m.ld2;
        }
    }
    // reg[4 ks + 2 q + p] = A[row p][32 c + 8 ks + t + 4 q]; indices past the contraction axis repeat the last one
    __device__ __forceinline__ void fetch(int c, float (&reg)[16]) const {
#pragma unroll
        for (int i = 0; i < 16; i++) {
            const int k = c * GKT + 8 * (i >> 2) + t + 4 * ((i >> 1) & 1);
            reg[i] = __ldg(base[i & 1] + (size_t)min(k, Kc - 1) * fld[i & 1]);
        }
    }
    __device__ __forceinline__ void split(int c, const float (&reg)[16], float (&hi)[16], float (&lo)[16]) const {
#pragma unroll
        for (int i = 0; i < 16; i++) {
            const int k = c * GKT + 8 * (i >> 2) + t + 4 * ((i >> 1) & 1);
            float v = one[i & 1] ? 1.f : reg[i];
            if (k >= Kc) v = 0.f;
            umma::split_tf32(v, hi[i], lo[i]);
        }
    }
};

template <int TN, bool BO, bool SWAP>
__global__ void __launch_bounds__(NLOAD, 1) k_gemm_ts(const GemmArgs g) {
    extern __shared__ __align__(128) unsigned char dsm[];
    constexpr int B_B = (TN / 8) * SBO, STAGE_B = 2 * B_B;
    const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31, z = blockIdx.z;
    const int a0 = blockIdx.x * TM, b0 = blockIdx.y * TN;
    const int nch = (g.Kc + GKT - 1) / GKT;
    const uint32_t base = umma::smem_u32(dsm);

    const FragA opA(g.A, z, a0, g.Mo, g.Kc);
    const Operand<TN, BO> opB(g.B, z, b0, g.No, g.Kc, w, lane);
    float ra[NSET][16], rb[NSET][TN / 32][4];
    float hi[16], lo[16], d[TN / 2];
#pragma unroll
    for (int p = 0; p < NSET - 1; p++)
        if (p < nch) { opA.fetch(p, ra[p]); opB.fetch(p, rb[p]); }
    for (int c0 = 0; c0 < nch; c0 += NSET) {
#pragma unroll
        for (int u = 0; u < NSET; u++) {
            const int c = c0 + u;
            if (c < nch) {
                if (c + NSET - 1 < nch) {
                    opA.fetch(c + NSET - 1, ra[(u + NSET - 1) % NSET]);
                    opB.fetch(c + NSET - 1, rb[(u + NSET - 1) % NSET]);
                }
                umma::wg_wait<0>();             // hi / lo are the operands of the previous chunk's products
                opA.split(c, ra[u], hi, lo);
                unsigned char *st = dsm + u * STAGE_B;
                opB.store(c, rb[u], st, st + B_B);
                umma::fence_async_smem();
                __syncthreads();
                const umma::Tile bh{base + u * STAGE_B, LBO, SBO}, bl = bh.shifted(B_B);
                umma::gemm3_rs<TN, GKT / 8>(d, hi, lo, bh, bl, c > 0);
                umma::wg_commit();
            }
        }
    }
    umma::wg_wait<0>();
    epilogue<TN, SWAP>(g, z, d, reinterpret_cast<float *>(dsm), a0, b0);
}

template <int TN>
constexpr int ts_smem_bytes() {
    constexpr int stages = NSTAGE * 2 * (TN / 8) * SBO, transpose = TM * (TN + 1) * 4;
    return stages > transpose ? stages : transpose;
}
template <int TN, bool BO, bool SWAP>
void launch_ts(const GemmArgs &g, int nets, cudaStream_t st) {
    dim3 grid((g.Mo + TM - 1) / TM, (g.No + TN - 1) / TN, nets);
    k_gemm_ts<TN, BO, SWAP><<<grid, NLOAD, ts_smem_bytes<TN>(), st>>>(g);
}

template <int TN>
constexpr int smem_bytes() { return NSTAGE * (2 * (TM / 8) * SBO + 2 * (TN / 8) * SBO); }

template <int TN, bool AO, bool BO>
cudaError_t prepare_one() {
    return cudaFuncSetAttribute(k_gemm_tc<TN, AO, BO>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes<TN>());
}

template <int TN, bool AO, bool BO>
void launch_one(const GemmArgs &g, int nets, cudaStream_t st) {
    dim3 grid((g.Mo + TM - 1) / TM, (g.No + TN - 1) / TN, nets);
    k_gemm_tc<TN, AO, BO><<<grid, NLOAD, smem_bytes<TN>(), st>>>(g);
}

template <bool AO, bool BO>
void launch_tn(const GemmArgs &g, int nets, cudaStream_t st, int tn) {
    if (tn == 64) launch_one<64, AO, BO>(g, nets, st);
    else launch_one<32, AO, BO>(g, nets, st);
}

}  // namespace

// >48 KB of dynamic shared memory needs the attribute; set once per device from prl_init (never inside a stream capture)
cudaError_t gemm_tc_prepare() {
    cudaError_t e;
    if ((e = prepare_one<64, true, true>()) != cudaSuccess) return e;
    if ((e = prepare_one<32, true, true>()) != cudaSuccess) return e;
    if ((e = prepare_one<64, true, false>()) != cudaSuccess) return e;
    if ((e = prepare_one<32, true, false>()) != cudaSuccess) return e;
    if ((e = prepare_one<64, false, false>()) != cudaSuccess) return e;
    if ((e = prepare_one<32, false, false>()) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(k_gemm_ts<64, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ts_smem_bytes<64>())) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(k_gemm_ts<32, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ts_smem_bytes<32>())) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(k_gemm_ts<64, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ts_smem_bytes<64>())) != cudaSuccess) return e;
    if ((e = cudaFuncSetAttribute(k_gemm_ts<32, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ts_smem_bytes<32>())) != cudaSuccess) return e;
    return cudaSuccess;
}

// engine: -1 = the library default (g_contraction_engine); 0 = SIMT tiles; 1 = automatic: tensor-core tiles from 4096 output
// rows on (see the header of this file), SIMT tiles below; 2 = tensor cores always (callers whose results must not depend
// on how many rows a launch sees: PPO's rollout passes); 64 / 32 = tensor cores with that tile width.
bool gemm_tc_launch(const GemmArgs &g, int nets, bool ao, bool bo, cudaStream_t st, int engine) {
    if (engine < 0) engine = g_contraction_engine;
    if (engine == 0 || g.Mo <= 0 || g.No <= 0 || g.Kc <= 0) return false;
    if (!ao && bo) return false;   // not a shape the learners use
    if (engine == 1 && g.Mo < 4096) return false;
    if (engine == 164 || engine == 132) engine = 2;    // the RS form declined the shape
    const int tn = engine == 64 || engine == 32 ? engine : (g.No > 32 ? 64 : 32);
    if (ao && bo) launch_tn<true, true>(g, nets, st, tn);
    else if (ao) launch_tn<true, false>(g, nets, st, tn);
    else launch_tn<false, false>(g, nets, st, tn);
    return true;
}

// RS form.  gs is already in the kernel's orientation: gs.A = the 128-row operand (its Mat rows are contracted), gs.Mo its
// extent, gs.B / gs.No the other operand; swap = the accumulator is C transposed.  Only on request (engine 164 / 132 = this
// form with tile width 64 / 32): the automatic choice uses the SS form, for which no learner has to keep transposed weights.
bool gemm_ts_launch(const GemmArgs &gs, int nets, bool bo, bool swap, cudaStream_t st, int engine) {
    if (engine < 0) engine = g_contraction_engine;
    if ((engine != 164 && engine != 132) || gs.Mo <= 0 || gs.No <= 0 || gs.Kc <= 0) return false;
    if (bo != swap) return false;   // the two combinations the learners use
    const int tn = engine == 164 ? 64 : 32;
    if (swap) { if (tn == 64) launch_ts<64, true, true>(gs, nets, st); else launch_ts<32, true, true>(gs, nets, st); }
    else { if (tn == 64) launch_ts<64, false, false>(gs, nets, st); else launch_ts<32, false, false>(gs, nets, st); }
    return true;
}

// dst[z][c][r] = src[z][r][c]  (the transposed weight copies the RS-form forward reads)
__global__ void k_transpose(int rows, int cols, const float *__restrict__ src, float *__restrict__ dst) {
    __shared__ float t[32][33];
    const size_t zo = (size_t)blockIdx.z * rows * cols;
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int y = threadIdx.y; y < 32; y += blockDim.y)
        if (r0 + y < rows && c0 + threadIdx.x < cols) t[y][threadIdx.x] = src[zo + (size_t)(r0 + y) * cols + c0 + threadIdx.x];
    __syncthreads();
    for (int y = threadIdx.y; y < 32; y += blockDim.y)
        if (c0 + y < cols && r0 + threadIdx.x < rows) dst[zo + (size_t)(c0 + y) * rows + r0 + threadIdx.x] = t[threadIdx.x][y];
}
void transpose_weights(int rows, int cols, int nets, const float *src, float *dst, cudaStream_t st) {
    dim3 grid((cols + 31) / 32, (rows + 31) / 32, nets), block(32, 8);
    k_transpose<<<grid, block, 0, st>>>(rows, cols, src, dst);
}

}  // namespace prl

extern "C" int prl_set_contraction_engine(int engine) {
    PRL_REQUIRE(engine >= 0 && engine <= 2, "engine must be 0 (SIMT tiles), 1 (automatic) or 2 (tensor-core tiles always)");
    prl::g_contraction_engine = engine;
    return PRL_OK;
}
extern "C" int prl_get_contraction_engine(void) { return prl::g_contraction_engine; }


// Test hook: one contraction of the learners' three kinds through GemmLauncher.
//   op 0  y[M x N]  = act(x W^T + b)          a = x [M x K] (or [M x split] with a2 = [M x (K - split)]), b = W [N x K]
//   op 1  dx[M x K] (+)= dy W  (masked)       a = dy [M x N], b = W [N x K], mask [M x K]
//   op 2  dW[N x K] = dy^T x, db = dy^T 1     a = dy [M x N], b = x [M x K] (or split with a2), c_tail = db [N]
// `nets` stacked problems are laid out contiguously in every operand.
extern "C" int prl_test_contraction(int op, int engine, int M, int N, int K, const float *a, const float *b, const float *a2, int split,
                                    const float *bias, const float *mask, int relu, int accumulate, float *c, float *c_tail, int nets,
                                    void *stream) {
    using namespace prl;
    PRL_REQUIRE(op >= 0 && op <= 2 && M > 0 && N > 0 && K > 0 && a && b && c && nets >= 1, "bad argument");
    GemmLauncher L;   // prl_init has prepared the kernels
    L.st = (cudaStream_t)stream;
    L.engine = engine;
    const long long MK = (long long)M * K, MN = (long long)M * N, NK = (long long)N * K;
    if (op == 0) {
        Mat X = a2 ? mat2(a, split, split, a2, K - split, (long long)M * split, (long long)M * (K - split)) : mat(a, K, MK);
        float *wt = nullptr;
        if (engine == 164 || engine == 132) {          // a learner using this form would keep the copy up to date itself
            PRL_CUDA(cudaMallocAsync((void **)&wt, sizeof(float) * NK * nets, L.st));
            transpose_weights(N, K, nets, b, wt, L.st);
        }
        L.fwd(X, M, b, K, NK, bias, N, N, K, relu != 0, c, N, MN, nets, wt, N, NK);
        if (wt) PRL_CUDA(cudaFreeAsync(wt, L.st));
    } else if (op == 1) {
        L.bwd_x(a, N, MN, M, N, b, K, NK, 0, K, c, K, MK, mask, K, MK, accumulate != 0, nets);
    } else {
        PRL_REQUIRE(c_tail, "op 2 needs c_tail");
        Mat X = a2 ? mat2(b, split, split, a2, K - split, (long long)M * split, (long long)M * (K - split)) : mat(b, K, MK);
        L.bwd_w(a, N, MN, M, N, X, K, c, K, NK, c_tail, N, nets);
    }
    PRL_CUDA(cudaGetLastError());
    return PRL_OK;
}
