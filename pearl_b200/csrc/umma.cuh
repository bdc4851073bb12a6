// umma.cuh — thin inline-PTX layer over Hopper's warpgroup tensor-core instruction
// (wgmma.mma_async, sm_90a) for the dense contractions of the learners.
//
// fp32 parity needs more than one TF32 pass: every fp32 operand x is split
//   x = hi + lo,  hi = trunc_tf32(x) (done by the hardware),  lo = x - hi
// and a product is accumulated as hi*hi + hi*lo + lo*hi in the fp32 register
// accumulator ("3xTF32"): relative error ~2^-21 per product instead of 2^-11.
//
// A product is issued by one whole warpgroup (128 threads, 4 consecutive warps):
// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, the accumulator spread over the warpgroup's registers:
//   thread (warp w of the warpgroup, g = lane / 4, t = lane % 4), register d[4 j + 2 p + e]
//   holds D[16 w + g + 8 p][8 j + 2 t + e]                                   (acc_row / acc_col below)
// B always comes from shared memory, A from shared memory (SS form) or from registers (RS form):
//   a[2 q + p] = A[16 w + g + 8 p][t + 4 q].
//
// Shared-memory operand tiles are in the canonical K-major NO-SWIZZLE ("interleaved") layout,
// written directly by SIMT code:
//   16-byte chunk c = k/4 of row r sits at  (r/8)*SBO + c*LBO + (r%8)*16
//   (8 rows x 16 B = one 128-byte core matrix; LBO = 128 B so the core matrices
//    of one 8-row group are contiguous along K; SBO = (K/4)*128 B)
// One wgmma of kind tf32 consumes K = 8 (two chunks); the next K step advances the
// descriptor start address by 2*LBO.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace umma {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- operand layout -------------------------------------------------------
constexpr int LBO = 128;  // bytes between the two 16-byte K chunks of one MMA / consecutive core matrices
__host__ __device__ constexpr int tile_sbo(int K) { return (K / 4) * 128; }           // bytes per 8-row group
__host__ __device__ constexpr int tile_bytes(int rows, int K) { return (rows / 8) * tile_sbo(K); }
// float index of element (r, k) inside a tile of K columns
__device__ __forceinline__ int tile_index(int r, int k, int K) {
    return (r >> 3) * (tile_sbo(K) >> 2) + (k >> 2) * 32 + (r & 7) * 4 + (k & 3);
}

// The tensor core TRUNCATES fp32 operands to TF32 (the 3xTF32 cases of tests/test_gpu_umma.py only reach 4e-6 if it
// does: with rounding, hi + lo would not add up to x), so the "hi" operand
// can be x itself and lo = x - trunc_tf32(x) (exact in fp32; its own truncation costs 2^-21 relative).
__device__ __forceinline__ float tf32_lo(float x) { return x - __uint_as_float(__float_as_uint(x) & 0xffffe000u); }
__device__ __forceinline__ void split_tf32(float x, float &hi, float &lo) {
    hi = x;
    lo = tf32_lo(x);
}

// ---- descriptors ------------------------------------------------------------
// shared-memory matrix descriptor: start address>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46),
// layout type [62,64) = 0 (no swizzle)
__device__ __forceinline__ uint64_t make_desc2(uint32_t smem_addr, int lbo_bytes, int sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3fff);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3fff) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3fff) << 32;
    return d;
}

// K-major operand tile with a free chunk pitch.  Element (r, k) of a tile with K columns lives at byte
//   (r/8)*sbo + (k/4)*lbo + (r%8)*16 + (k%4)*4,   sbo = (K/4)*lbo.
// lbo = 128: dense (rows written by their owner thread as 16-byte chunks);
// lbo = 144: "transposed-write friendly": when 32 lanes write the SAME row r and consecutive k
//            (a thread that owns batch row k scatters its values into column k of the tile), the
//            addresses (k/4)*144 + (k%4)*4 hit 32 distinct banks.
// wgmma has no MN-major form for tf32 operands, so the backward pass builds explicitly transposed tiles.
struct Tile {
    uint32_t addr;  // shared-memory byte address
    int lbo, sbo;   // bytes
    // The descriptor of K step `kstep`, built from the 32-bit address right where its wgmma is issued.  The address passes
    // through an empty volatile asm, so the compiler cannot hoist the descriptors out of the loops around a product and
    // keep every K step's 64-bit descriptor live (and spilled) across a whole kernel.
    __device__ __forceinline__ uint64_t desc(int kstep) const {
        uint32_t a = addr;
        asm volatile("" : "+r"(a));
        return make_desc2(a + (uint32_t)kstep * 2 * lbo, lbo, sbo);
    }
    __device__ __forceinline__ Tile rows_from(int r) const { return Tile{addr + (uint32_t)(r >> 3) * sbo, lbo, sbo}; }  // r % 8 == 0
    __device__ __forceinline__ Tile shifted(uint32_t bytes) const { return Tile{addr + bytes, lbo, sbo}; }
};
__host__ __device__ constexpr int tile_bytes2(int rows, int K, int lbo) { return (rows / 8) * (K / 4) * lbo; }
__device__ __forceinline__ int tile_index2(int r, int k, int K, int lbo) {
    return (r >> 3) * ((K >> 2) * (lbo >> 2)) + (k >> 2) * (lbo >> 2) + (r & 7) * 4 + (k & 3);
}
__device__ __forceinline__ Tile make_tile(const void *p, int K, int lbo) { return Tile{smem_u32(p), lbo, (K >> 2) * lbo}; }

// ---- accumulator / register-operand coordinates of this thread -----------------
__device__ __forceinline__ int acc_row(int p) { return ((threadIdx.x >> 5) & 3) * 16 + ((threadIdx.x & 31) >> 2) + 8 * p; }  // p = 0, 1
__device__ __forceinline__ int acc_col(int j, int e) { return 8 * j + 2 * (threadIdx.x & 3) + e; }                            // e = 0, 1
// A product whose A operand is a previous accumulator (RS form) contracts over the accumulator's columns: K slot t of
// step j is fed from column 8 j + 2 t and slot t + 4 from column 8 j + 2 t + 1.  The B tile of such a product stores
// column k of its matrix at the K position kperm(k), which makes the pairing right without moving a register.
__host__ __device__ constexpr int kperm(int k) { return (k & ~7) | ((k & 1) << 2) | ((k & 7) >> 1); }

// ---- synchronisation of the asynchronous tensor-core proxy -------------------------
// registers written by ordinary instructions (accumulators, RS operands) -> visible to the next wgmma
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }
// make generic-proxy shared-memory writes visible to the tensor core (async proxy)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- one wgmma: D[64 x N] (+)= A[64 x 8] B[N x 8]^T, N in {8, 16, 32, 64}; d: N / 2 registers -----------
template <int N> struct Mma;

#define UMMA_D4(o) "+f"(d[o]), "+f"(d[o + 1]), "+f"(d[o + 2]), "+f"(d[o + 3])
#define UMMA_D8(o) UMMA_D4(o), UMMA_D4(o + 4)
#define UMMA_D16(o) UMMA_D8(o), UMMA_D8(o + 8)
#define UMMA_D32(o) UMMA_D16(o), UMMA_D16(o + 16)
#define UMMA_DEFINE(N, DREGS, DOPS, A0, B0, P0)                                                                         \
    template <> struct Mma<N> {                                                                                         \
        static __device__ __forceinline__ void ss(float *d, uint64_t a_desc, uint64_t b_desc, bool accumulate) {        \
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #P0 ", 0;\n\t"                                        \
                         "wgmma.mma_async.sync.aligned.m64n" #N "k8.f32.tf32.tf32 " DREGS ", %" #A0 ", %" #B0 ", p, 1, 1;\n\t}\n" \
                         : DOPS                                                                                         \
                         : "l"(a_desc), "l"(b_desc), "r"((uint32_t)accumulate));                                        \
        }                                                                                                               \
    };
UMMA_DEFINE(8, "{%0, %1, %2, %3}", UMMA_D4(0), 4, 5, 6)
UMMA_DEFINE(16, "{%0, %1, %2, %3, %4, %5, %6, %7}", UMMA_D8(0), 8, 9, 10)
UMMA_DEFINE(32, "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}", UMMA_D16(0), 16, 17, 18)
UMMA_DEFINE(64,
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
            "%24, %25, %26, %27, %28, %29, %30, %31}",
            UMMA_D32(0), 32, 33, 34)
#undef UMMA_DEFINE

// RS form (A fragment a[0..3] in registers), N in {32, 64}
template <int N>
__device__ __forceinline__ void mma_rs(float *d, const float *a, uint64_t b_desc, bool accumulate);
template <>
__device__ __forceinline__ void mma_rs<32>(float *d, const float *a, uint64_t b_desc, bool accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}\n"
                 : UMMA_D16(0)
                 : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
                   "l"(b_desc), "r"((uint32_t)accumulate));
}
template <>
__device__ __forceinline__ void mma_rs<64>(float *d, const float *a, uint64_t b_desc, bool accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
                 "%24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}\n"
                 : UMMA_D32(0)
                 : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])),
                   "l"(b_desc), "r"((uint32_t)accumulate));
}
#undef UMMA_D32
#undef UMMA_D16
#undef UMMA_D8
#undef UMMA_D4

// 3xTF32, SS form: d[64 x N] (+)= A[64 x K] * B[N x K]^T; executed by every thread of ONE warpgroup, which must have
// fenced its shared-memory writes (fence_async_smem + barrier) before.  *_exact: the operand is exactly representable in
// TF32 (0/1 indicators), its lo tile is not needed.  Each wgmma gets its descriptors from Tile::desc.  The caller commits
// and waits (wg_commit / wg_wait).
template <int N>
__device__ __forceinline__ void gemm3(float *d, Tile a_hi, Tile a_lo, Tile b_hi, Tile b_lo, int K, bool accumulate_first,
                                      bool a_exact = false, bool b_exact = false) {
    bool acc = accumulate_first;
    wg_fence();
    for (int ks = 0; ks < (K >> 3); ks++) {
        if (!a_exact) { Mma<N>::ss(d, a_lo.desc(ks), b_hi.desc(ks), acc); acc = true; }   // small terms first
        if (!b_exact) { Mma<N>::ss(d, a_hi.desc(ks), b_lo.desc(ks), acc); acc = true; }
        Mma<N>::ss(d, a_hi.desc(ks), b_hi.desc(ks), acc);
        acc = true;
    }
}

// 3xTF32, RS form: a_hi / a_lo hold this thread's A fragments of (at most) KSTEPS K steps (4 registers each).  The registers
// must not be written again before the products have been waited for.  A runtime ksteps < KSTEPS puts a branch into the
// chain, and ptxas then serialises every wgmma of the kernel: pipelined kernels leave it at KSTEPS.
// B_LO_FIRST issues a_hi*b_lo before a_lo*b_hi: the small terms in the order gemm3 adds them for the transposed product
// (B^T A^T), so that computing a transpose this way gives the same bits.
template <int N, int KSTEPS, bool B_LO_FIRST = false>
__device__ __forceinline__ void gemm3_rs(float *d, const float *a_hi, const float *a_lo, Tile b_hi, Tile b_lo, bool accumulate_first,
                                         int ksteps = KSTEPS) {
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < KSTEPS; ks++) {
        if (ks >= ksteps) break;
        if (B_LO_FIRST) {
            mma_rs<N>(d, a_hi + 4 * ks, b_lo.desc(ks), accumulate_first || ks > 0);
            mma_rs<N>(d, a_lo + 4 * ks, b_hi.desc(ks), true);
        } else {
            mma_rs<N>(d, a_lo + 4 * ks, b_hi.desc(ks), accumulate_first || ks > 0);
            mma_rs<N>(d, a_hi + 4 * ks, b_lo.desc(ks), true);
        }
        mma_rs<N>(d, a_hi + 4 * ks, b_hi.desc(ks), true);
    }
}

// ---- mbarrier (completion of TMA bulk copies) -------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// Bounded spin: a wait that cannot complete (protocol bug, lost TMA transaction) ends the kernel with a trap instead of
// hanging the device — over a second of polling, orders of magnitude beyond any legitimate wait.  No printf here: a
// function call anywhere in a kernel makes ptxas serialise every wgmma of that kernel (warning C7510).
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    const uint32_t a = smem_u32(bar);
    uint32_t done;
    long long t0 = 0;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.b32 %0, 1, 0, p;\n\t}\n"
            : "=r"(done)
            : "r"(a), "r"(parity)
            : "memory");
        if (!done) {
            if (t0 == 0) t0 = clock64();
            if (clock64() - t0 < 3000000000ll) continue;   // ~1.5 s of SM clocks
            __trap();
        }
    } while (!done);
}

}  // namespace umma
