// Conv2D (1x1 and k x k, stride 1 and 2) as an implicit GEMM on Hopper's tensor cores, hand-written for sm_90a: TMA
// (cp.async.bulk.tensor) stages NHWC activation tiles and packed weights from HBM into 128B-swizzled shared memory, two
// consumer warpgroups run wgmma.mma_async on them with fp32 accumulators in registers and then the epilogue of their rows
// (bias + residual + activation + split-fp16, staged in swizzled shared memory and written with one TMA store per slab).
//
//   D[M = 128 output pixels, N = n_blk <= 128 output channels] += A[M, K] * B[N, K]^T,   K = (tap, 64-channel block)
//
// fp32-faithful arithmetic out of fp16 tensor cores: activations and weights are stored as hi + lo fp16 pairs
// (snnb_internal.h); the product terms of one K block (one ring stage) accumulate into a fresh fp32 accumulator, which is then
// added to the tile's fp32 sum (acc_promote). Template parameter TERMS:
//   3:  A_hi*B_hi + A_hi*B_lo + A_lo*B_hi  (the dropped A_lo*B_lo term is ~2^-24 relative): ~22 mantissa bits per operand.
//   2:  (A_hi + A_lo) * B_hi: the weights rounded ONCE to fp16 (<= 2^-12 relative per weight, per-layer error vs the oracle
//       ~1e-4 of the tensor's range - inside the 1e-3 budget).
//   1:  A_hi * B_hi: the half-precision storage mode (the reference's RGBA16F), no lo planes anywhere.
//
// A tile = a (tw x th x tn)-pixel box of the OUTPUT grid (tw*th*tn <= 128): for filter tap (ky,kx) the producer issues
// ONE 4-D TMA box load at input coordinate (ox0*s + kx - pad_x, oy0*s + ky - pad_y); out-of-range rows/columns are
// zero-filled by the TMA unit, which is exactly the reference's constant padding (vk_conv2d.comp:168-172), and the
// channel tail (c >= IC) is zero-filled too, so no im2col buffer and no boundary code exist anywhere.
//
// Roles (384 threads, persistent CTAs, one per SM): warpgroup 0 = TMA producer (one thread issues the operand loads, one thread
// of warp 1 the epilogue's residual loads and output stores), warpgroups 1 and 2 = consumers, each owning 64 of the tile's 128
// rows: one m64 wgmma per K step and product term, issued in turns with the other consumer, then the epilogue arithmetic of
// those rows. The operand ring (full/empty mbarriers) is as deep as shared memory allows for the launch's n_blk, so the producer
// runs several K blocks ahead. Layers with few tiles split K over several CTAs (fp32 partials, last arriver reduces), or,
// on request, use a stream-K decomposition. Also in this file: the row-window kernel for small-channel stems and the
// TMA-staged depthwise kernel.
//
// Reference semantics: shadertemplate_vk_conv2d.comp:148-347, vk_conv2d_1x1.comp:68-211 (+ fused vk_add.comp:41-90).
#include <cuda.h>

#include <algorithm>
#include <vector>

#include "snnb_internal.h"

namespace snnb {

// UM_BLOCK_M, UM_BLOCK_K, UM_MAX_N, UM_STG_BYTES, UM_SMEM_LIMIT and the RW_* limits the planner reads are in snnb_internal.h
constexpr int UM_A_BYTES     = UM_BLOCK_M * 128;
constexpr int UM_CONSUMERS   = 2;                          // consumer warpgroups, 64 tile rows each
constexpr int UM_THREADS     = 128 * (1 + UM_CONSUMERS);   // warpgroup 0 = producer
constexpr int UM_EPI_THREADS = 128 * UM_CONSUMERS;
constexpr int UM_BAR_BYTES   = 256;
constexpr int UM_TURN_BAR    = 1;                          // named barriers 1, 2: consumer warpgroup 1's / 2's turn to issue (0 = __syncthreads)

// Shared-memory carve-up of conv_umma_kernel<TERMS, NB>: [ring: STAGES x (A_hi, A_lo, B_hi, B_lo)] [staging] [barriers]. A stage
// holds only the planes the product reads, and the ring takes whatever shared memory the staging buffer leaves (at most 8 stages).
template <int TERMS, int NB> struct UmGeom {
    static constexpr int A_PLANES    = TERMS == 1 ? 1 : 2;
    static constexpr int B_PLANES    = TERMS == 3 ? 2 : 1;
    static constexpr int B_BYTES     = NB * 128; // one plane: NB rows of 64 K columns (a multiple of 1024 B: SWIZZLE_128B alignment)
    static constexpr int STAGE_BYTES = A_PLANES * UM_A_BYTES + B_PLANES * B_BYTES;
    static constexpr int FIT         = (UM_SMEM_LIMIT - 1024 - UM_BAR_BYTES - UM_STG_BYTES) / STAGE_BYTES;
    static constexpr int STAGES      = FIT > 8 ? 8 : FIT;
    static constexpr int SMEM_BYTES  = STAGES * STAGE_BYTES + UM_STG_BYTES + 1024 /*alignment slack*/ + UM_BAR_BYTES;
    static_assert(STAGES >= 2, "operand ring needs two stages");
};

struct UmmaParams {
    const float* bias;
    int N, OH, OW, OC, OCp;
    int tw, th, tn, rows_used;
    int tiles_x, tiles_y, tiles_n, tiles_oc, n_blk;
    int ksize, stride, pad_x, pad_y;
    int cblocks, ICp;
    int act;
    float alpha;
    int has_res;
    // split-K (layers with too few output tiles to fill the GPU, e.g. 7x7x512): work item = (tile, K range). Every item
    // dumps its fp32 partial tile to `partials`, bumps the tile's arrival counter, and the LAST arriver sums all partials
    // in split order (deterministic) and runs the normal epilogue.
    int ksplit, kb_per_split;
    float* partials; // [tile][split][128 rows][n_blk]
    int* counters;   // [tile], zero between launches (the last arriver resets it)
    int has_lo;      // the output tensor has a lo plane (0 in the fp16 storage mode)
    // Stream-K (sk != 0): the first sk_dp tiles (a multiple of the grid) are whole-tile work items, CTA b taking tiles
    // b, b + grid, ...; the K-block units of the remaining tiles (sk_units = tiles x K blocks, laid end to end) are cut into sk_ctas
    // equal ranges, CTA b < sk_ctas taking range b - which covers the tail of one tile and the head of the next. A tile cut into
    // pieces is finished like a split-K tile (fp32 partials, last arriver sums them in piece order). Work ids: [0, sk_dp) tiles,
    // sk_dp + 4 c + j = the j-th piece of CTA c's range; the schedule is static: pieces first, then tiles.
    int sk, sk_dp, sk_ctas;
    long long sk_units;
};

// ---------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t) __cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a broken descriptor or protocol bug must surface as a trapped kernel, never as a hung GPU (SNNB_SYNC_LAYERS=1
// names the layer and kernel that trapped). It must not make a function call (no printf): ptxas serializes every wgmma of a kernel
// that contains a call, each one waiting for the previous one to retire.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity))
        if (clock64() - t0 > 4000000000LL) __trap();
}
// One lane of a CONVERGED warp: the compiler knows a single thread is active in the guarded region, so the TMA issue is
// one predicated instruction rather than a loop over the active lanes.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) { asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory"); }
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(dst), "l"(m),
                 "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                 : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(dst), "l"(m), "r"(bar),
                 "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst), "l"(m), "r"(bar),
                 "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(m), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                 : "memory");
}
// plain (non-tensor) bulk copy global -> shared, completion on an mbarrier; 16-byte aligned addresses and size
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// L2 prefetch of a tensor box (no shared memory, no completion to wait for)
__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap* m, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile [%0, {%1, %2, %3, %4}];" ::"l"(m), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
__device__ __forceinline__ void named_bar_arrive(int id, int threads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// wgmma shared-memory matrix descriptor (sm_90), K-major operand, SWIZZLE_128B:
//   [0,14) start address >> 4 | [16,30) LBO >> 4 (= 1, unused for swizzled K-major) | [32,46) SBO >> 4 (= 1024 B: 8 rows x 128 B)
//   [62,64) layout type = 1 (SWIZZLE_128B). A K step of 16 fp16 (32 B) inside the 128-byte row adds 2 to the address field.
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t saddr) {
    return (uint64_t) ((saddr >> 4) & 0x3FFFu) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// Un-swizzled K-major descriptor with an overlapping K stride (row-window kernel): LBO = 16 B (next 16-byte K chunk = next
// pixel), SBO = 128 B (8 rows x 16 B), layout type 0.
__device__ __forceinline__ uint64_t gmma_desc_window(uint32_t saddr) { return (uint64_t) ((saddr >> 4) & 0x3FFFu) | (1ull << 16) | (8ull << 32); }

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x N] (fp32 registers) (+)= A[64 x 16] * B[N x 16]^T, both fp16 K-major operands in shared memory, issued by a whole
// warpgroup; accumulate = 0 overwrites D. Fragment of thread t (warp w = t / 32 of the warpgroup, lane l): d[4 j + 2 r + b] = D[16 w + l / 4 + 8 r][8 j + 2 (l % 4) + b].
template <int N> struct Wgmma;
template <> struct Wgmma<32> {
    static __device__ __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t accumulate) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                     : "l"(a), "l"(b), "r"(accumulate));
    }
};
template <> struct Wgmma<64> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "l"(a), "l"(b), "r"(accumulate));
    }
};
template <> struct Wgmma<128> {
    static __device__ __forceinline__ void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t accumulate) {
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                     "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                     : "l"(a), "l"(b), "r"(accumulate));
    }
};

template <int NACC> __device__ __forceinline__ void acc_fence(float (&d)[NACC]) {
#pragma unroll
    for (int i = 0; i < NACC; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Two-level accumulation: every K block (every ring stage) is summed by the tensor core into a FRESH accumulator, which is then
// added to the tile's fp32 sum with round-to-nearest FADDs. The tensor core's own accumulation chain is thus one K block long
// whatever the layer's K, and a tile's result does not depend on how its K range was split over CTAs beyond the order in which
// whole-block sums are added.
template <int NACC> __device__ __forceinline__ void acc_promote(float (&sum)[NACC], float (&d)[NACC]) {
    acc_fence(d);
#pragma unroll
    for (int i = 0; i < NACC; ++i) sum[i] += d[i];
}
__device__ __forceinline__ void regs_dealloc_40() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void regs_alloc_232() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }

// transcendental activations (tanh / sigmoid / SiLU). Inlined into the tensor-core kernels: a call would serialize their wgmmas.
__device__ __forceinline__ float umma_act(float v, int act, float alpha) {
    switch (act) {
    case SNNB_ACT_RELU: return fmaxf(v, 0.0f);
    case SNNB_ACT_RELU6: return fminf(fmaxf(v, 0.0f), 6.0f);
    case SNNB_ACT_TANH: return tanhf(v);
    case SNNB_ACT_SIGMOID: return 1.0f / (1.0f + expf(-v));
    case SNNB_ACT_LEAKY_RELU: return fmaxf(v, v * alpha);
    case SNNB_ACT_SILU: return v * 1.0f / (1.0f + expf(-v));
    default: return v;
    }
}
// out of line for the depthwise kernel, which issues no wgmma: its hot loop stays small
__device__ __noinline__ float umma_act_call(float v, int act, float alpha) { return umma_act(v, act, alpha); }
// split-fp16 (snnb_internal.h): packed pair conversions, round to nearest, saturated to +-65504
__device__ __forceinline__ float2 um_h2f(uint32_t u) { return __half22float2(*reinterpret_cast<const __half2*>(&u)); }
__device__ __forceinline__ uint32_t um_f2h(float a, float b) {
    uint32_t h;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(b), "f"(a));
    return h;
}
__device__ __forceinline__ void um_split2(float a, float b, uint32_t& h, uint32_t& l) {
    h               = um_f2h(a, b);
    const float2 hf = um_h2f(h);
    l               = um_f2h(a - hf.x, b - hf.y);
}

// ---------------------------------------------------------------------------------------------------------------
// Epilogue of one output tile, shared by both tensor-core kernels: accumulator registers -> +bias (+residual) -> activation ->
// split-fp16 -> SHARED MEMORY (128B-swizzled for full 64-channel slabs) -> ONE TMA bulk store per plane and slab. The TMA store
// writes full 128-byte lines and clips rows / channels that fall outside the tensor by itself. The fused residual (Conv2D -> Add)
// comes in the same way: a TMA box load of the residual slab into the staging buffer, read back by each thread at exactly the
// place it then overwrites.
//
// Each consumer warpgroup runs the arithmetic of its own 64 rows (disjoint in the staging buffer) on its own schedule; all TMA
// traffic of the epilogue belongs to one STORE THREAD in the producer warpgroup, which walks the same work list. Per slab, two
// mbarriers hand the staging buffer back and forth:
//   stg_ready (1 arrival + residual bytes): the previous slab's store has read the buffer out, and this slab's residual (if any)
//            has landed in it. The store thread arms it as soon as the buffer is free, so the residual load runs under the
//            consumers' K loop rather than between their K loop and their arithmetic.
//   stg_full  (one arrival per consumer thread): both warpgroups' rows are written; the store thread issues the slab's stores and
//            waits for them to read the buffer out.
// No consumer thread ever waits for a store.
// ---------------------------------------------------------------------------------------------------------------
struct EpiArgs {
    const CUtensorMap *o_hi64, *o_lo64, *o_hiT, *o_loT; // output maps: 64-channel slab (SWIZZLE_128B) and narrow slab (dense)
    const CUtensorMap *r_hi64, *r_lo64, *r_hiT, *r_loT; // residual maps, same geometry
    const float* bias;
    int OC, act, has_res, rows_box;
    int has_lo;          // write (and read, for the residual) the lo plane; 0 in the fp16 storage mode
    float alpha;
    uint32_t stg;        // staging smem (hi plane; lo plane at + UM_BLOCK_M * 128)
    uint32_t stg_ready;  // mbarrier: staging free (and the residual slab loaded)
    uint32_t stg_full;   // mbarrier: staging written by every consumer thread
};

// Store thread's side of one tile's epilogue: (oc0, c1, c2, c3) = the tile's box in the output (and residual) tensor. The staging
// buffer is free on entry (every earlier store has been read out) and again on return.
template <int NB>
__device__ __forceinline__ void epilogue_store_tile(const EpiArgs& e, int oc0, int c1, int c2, int c3, uint32_t& full_phase) {
    constexpr int W          = NB < 64 ? NB : 64;
    constexpr bool SW        = W == 64;
    constexpr uint32_t PITCH = SW ? 128u : (uint32_t) W * 2u;
    const uint32_t lo_off    = UM_BLOCK_M * 128;
    if (e.has_res) // the later slabs' residual, from L2 when their turn comes
        for (int sl = 1; sl < NB / W; ++sl) {
            tma_prefetch_4d(e.r_hi64, oc0 + sl * 64, c1, c2, c3);
            if (e.has_lo) tma_prefetch_4d(e.r_lo64, oc0 + sl * 64, c1, c2, c3);
        }
    for (int sl = 0; sl < NB / W; ++sl) {
        if (e.has_res) {
            mbar_expect_tx(e.stg_ready, (e.has_lo ? 2u : 1u) * (uint32_t) e.rows_box * PITCH);
            tma_load_4d(e.stg, SW ? e.r_hi64 : e.r_hiT, e.stg_ready, oc0 + sl * 64, c1, c2, c3);
            if (e.has_lo) tma_load_4d(e.stg + lo_off, SW ? e.r_lo64 : e.r_loT, e.stg_ready, oc0 + sl * 64, c1, c2, c3);
        } else {
            mbar_arrive(e.stg_ready);
        }
        mbar_wait(e.stg_full, full_phase);
        full_phase ^= 1u;
        tma_store_4d(SW ? e.o_hi64 : e.o_hiT, e.stg, oc0 + sl * 64, c1, c2, c3);
        if (e.has_lo) tma_store_4d(SW ? e.o_lo64 : e.o_loT, e.stg + lo_off, oc0 + sl * 64, c1, c2, c3);
        bulk_commit();
        bulk_wait_read0();
    }
}

// Consumer warpgroup's side. acc: this thread's fragment of its warpgroup's 64 x NB accumulator; row0 = the tile row of its d[0]
// (16 w + l / 4 within the warpgroup's rows), q = l % 4. SLOW_ACT: the activation is not one of the piecewise-linear ones (umma_act).
template <int NB, bool SLOW_ACT>
__device__ __forceinline__ void epilogue_tile_act(const EpiArgs& e, const float (&acc)[NB / 2], int oc0, int row0, int q, uint32_t& ready_phase) {
    constexpr int W      = NB < 64 ? NB : 64; // slab width in channels
    constexpr bool SW    = W == 64;            // full slab: 128-byte rows, SWIZZLE_128B
    constexpr uint32_t PITCH = SW ? 128u : (uint32_t) W * 2u;
    const float slope    = (e.act == SNNB_ACT_RELU || e.act == SNNB_ACT_RELU6) ? 0.0f : (e.act == SNNB_ACT_LEAKY_RELU ? e.alpha : 1.0f);
    const float hi_clip  = e.act == SNNB_ACT_RELU6 ? 6.0f : __int_as_float(0x7f800000);
    const uint32_t lo_off = UM_BLOCK_M * 128;
#pragma unroll
    for (int sl = 0; sl < NB / W; ++sl) {
        mbar_wait(e.stg_ready, ready_phase);
        ready_phase ^= 1u;
#pragma unroll
        for (int j = 0; j < W / 8; ++j) {
            const int c = sl * 64 + 8 * j + 2 * q; // channel of the pair within the tile
            const int oc = oc0 + c;
            const float b0 = oc < e.OC ? __ldg(e.bias + oc) : 0.0f, b1 = oc + 1 < e.OC ? __ldg(e.bias + oc + 1) : 0.0f;
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const int row = row0 + 8 * r;
                const uint32_t a = e.stg + (uint32_t) row * PITCH + (SW ? ((((uint32_t) j) ^ (uint32_t) (row & 7)) << 4) : (uint32_t) j * 16u) + (uint32_t) q * 4u;
                float v0 = acc[(sl * 8 + j) * 4 + 2 * r] + b0, v1 = acc[(sl * 8 + j) * 4 + 2 * r + 1] + b1;
                if (e.has_res) {
                    uint32_t hh, ll = 0u;
                    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(hh) : "r"(a));
                    if (e.has_lo) asm volatile("ld.shared.b32 %0, [%1];" : "=r"(ll) : "r"(a + lo_off));
                    const float2 rh = um_h2f(hh), rl = um_h2f(ll);
                    v0 += rh.x + rl.x;
                    v1 += rh.y + rl.y;
                }
                if (SLOW_ACT) {
                    v0 = umma_act(v0, e.act, e.alpha), v1 = umma_act(v1, e.act, e.alpha);
                } else if (e.act == SNNB_ACT_RELU) {
                    v0 = fmaxf(v0, 0.0f), v1 = fmaxf(v1, 0.0f);
                } else if (e.act != SNNB_ACT_NONE) {
                    v0 = fminf(fmaxf(v0, v0 * slope), hi_clip), v1 = fminf(fmaxf(v1, v1 * slope), hi_clip);
                }
                if (oc >= e.OC) v0 = 0.0f; // channels [OC, Cp) stay zero
                if (oc + 1 >= e.OC) v1 = 0.0f;
                uint32_t h, l;
                um_split2(v0, v1, h, l);
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(h) : "memory");
                if (e.has_lo) asm volatile("st.shared.b32 [%0], %1;" ::"r"(a + lo_off), "r"(l) : "memory");
            }
        }
        fence_async_smem(); // generic-proxy smem writes -> visible to the TMA (async proxy)
        mbar_arrive(e.stg_full); // by every thread: a lane-0 arrive is a divergent branch that makes ptxas serialize some kernels' wgmmas
    }
}

// The transcendental activations get an epilogue of their own, chosen once per tile: inlined into every element of the unrolled loop
// (the kernel makes no calls), their code would be strewn through the common epilogue's and more than double its size.
template <int NB>
__device__ __forceinline__ void epilogue_tile(const EpiArgs& e, const float (&acc)[NB / 2], int oc0, int row0, int q, uint32_t& ready_phase) {
    if (e.act == SNNB_ACT_NONE || e.act == SNNB_ACT_RELU || e.act == SNNB_ACT_RELU6 || e.act == SNNB_ACT_LEAKY_RELU)
        epilogue_tile_act<NB, false>(e, acc, oc0, row0, q, ready_phase);
    else
        epilogue_tile_act<NB, true>(e, acc, oc0, row0, q, ready_phase);
}

// After the store thread's last tile: its bulk stores must have completed before the CTA (and its shared memory) goes away.
__device__ __forceinline__ void epilogue_drain() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------------------------
// The kernel
// ---------------------------------------------------------------------------------------------------------------
// One work item of conv_umma_kernel: which tile, which K blocks, and - when the tile's K range is shared between CTAs - which piece
// of how many, plus the slot of its partial tiles.
struct WorkItem {
    int tile, kb0, kb1, piece, pieces, slot;
};
template <bool SK> // compile-time: the stream-K arithmetic (64-bit divisions) stays out of every other instantiation
__host__ __device__ __forceinline__ WorkItem decode_work(const UmmaParams& p, int work, int total_tiles, int num_kb) {
    WorkItem w;
    if constexpr (!SK) {
        const int split = work / total_tiles;
        w.tile = work - split * total_tiles, w.kb0 = split * p.kb_per_split, w.kb1 = w.kb0 + p.kb_per_split < num_kb ? w.kb0 + p.kb_per_split : num_kb;
        w.piece = split, w.pieces = p.ksplit, w.slot = w.tile;
    } else if (work < p.sk_dp) {
        w.tile = work, w.kb0 = 0, w.kb1 = num_kb, w.piece = 0, w.pieces = 1, w.slot = 0;
    } else {
        const int c = (work - p.sk_dp) >> 2, j = (work - p.sk_dp) & 3;
        const long long b0 = (long long) c * p.sk_units / p.sk_ctas, b1 = (long long) (c + 1) * p.sk_units / p.sk_ctas; // this CTA's units
        const int jt = (int) (b0 / num_kb) + j; // tile (counted from sk_dp) of the CTA's j-th piece
        const long long t0 = (long long) jt * num_kb, t1 = t0 + num_kb;
        w.tile = p.sk_dp + jt, w.slot = jt;
        w.kb0 = (int) ((b0 > t0 ? b0 : t0) - t0), w.kb1 = (int) ((b1 < t1 ? b1 : t1) - t0);
        // CTA holding unit u: ((u + 1) * ctas - 1) / units
        const int c_first = (int) (((t0 + 1) * p.sk_ctas - 1) / p.sk_units), c_last = (int) ((t1 * p.sk_ctas - 1) / p.sk_units);
        w.piece = c - c_first, w.pieces = c_last - c_first + 1;
    }
    return w;
}
// Static schedule of a stream-K launch: CTA `cta` first works off the pieces of its K-block range, then its whole tiles cta, cta + grid, ...
// (pieces first: a cut tile's last arriver sums the partials while the other CTAs are busy with whole tiles, not at the very end of the
// launch with everybody waiting). Returns the work id after `work` (`end` when there is none) / the first one.
__host__ __device__ __forceinline__ int sk_next_work(const UmmaParams& p, int work, int cta, int grid, int num_kb, int end) {
    if (work < p.sk_dp) return work + grid < p.sk_dp ? work + grid : end;
    const int c = (work - p.sk_dp) >> 2, j = ((work - p.sk_dp) & 3) + 1;
    const long long b0 = (long long) c * p.sk_units / p.sk_ctas, b1 = (long long) (c + 1) * p.sk_units / p.sk_ctas;
    if (j < 4 && b0 / num_kb + j <= (b1 - 1) / num_kb) return work + 1;
    return cta < p.sk_dp ? cta : end;
}
__host__ __device__ __forceinline__ int sk_first_work(const UmmaParams& p, int cta, int end) {
    return cta < p.sk_ctas ? p.sk_dp + 4 * cta : (cta < p.sk_dp ? cta : end);
}

// TERMS: how the fp32-faithful product is formed (see the top of the file). NB: output channels per tile (= UmmaParams::n_blk).
// SK: stream-K work decomposition (UmmaParams::sk); otherwise CTA b takes work items b, b + grid, ...
template <int TERMS, int NB, bool SK>
__global__ void __launch_bounds__(UM_THREADS, 1)
conv_umma_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo, const __grid_constant__ CUtensorMap tmB_hi,
                 const __grid_constant__ CUtensorMap tmB_lo, const __grid_constant__ CUtensorMap tmO_hi64, const __grid_constant__ CUtensorMap tmO_lo64,
                 const __grid_constant__ CUtensorMap tmO_hiT, const __grid_constant__ CUtensorMap tmO_loT, const __grid_constant__ CUtensorMap tmR_hi64,
                 const __grid_constant__ CUtensorMap tmR_lo64, const __grid_constant__ CUtensorMap tmR_hiT, const __grid_constant__ CUtensorMap tmR_loT,
                 const UmmaParams p) {
    using G = UmGeom<TERMS, NB>;
    constexpr int STAGES = G::STAGES;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u; // SWIZZLE_128B tiles need 1024-byte alignment
    const uint32_t stg       = smem_base + STAGES * G::STAGE_BYTES;
    const uint32_t bar_base  = stg + UM_STG_BYTES;
    // barrier slots (8 bytes each): full[0..S), empty[S..2S), staging ready / full, split-K partials dumped / verdict, split-K
    // "arrived last" flag
    auto full_bar  = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
    const uint32_t stg_ready   = bar_base + 8u * (2 * STAGES);
    const uint32_t stg_full    = bar_base + 8u * (2 * STAGES + 1);
    const uint32_t dumped_bar  = bar_base + 8u * (2 * STAGES + 2);
    const uint32_t verdict_bar = bar_base + 8u * (2 * STAGES + 3);
    const uint32_t last_flag   = bar_base + 8u * (2 * STAGES + 4);
    static_assert(8 * (2 * STAGES + 5) <= UM_BAR_BYTES, "barrier area");

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    pdl_trigger(); // the next kernel may start launching; it waits for this grid's completion before touching memory
    if (threadIdx.x == 0) {
        mbar_init(stg_ready, 1);
        mbar_init(stg_full, UM_EPI_THREADS);
        mbar_init(dumped_bar, UM_EPI_THREADS);
        mbar_init(verdict_bar, 1);
        tma_prefetch_desc(&tmA_hi);
        tma_prefetch_desc(&tmA_lo);
        tma_prefetch_desc(&tmB_hi);
        tma_prefetch_desc(&tmB_lo);
        tma_prefetch_desc(&tmO_hi64);
        tma_prefetch_desc(&tmO_lo64);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), UM_EPI_THREADS / 32); // one arrive per consumer warp
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait(); // barrier set-up and tensor-map prefetch overlapped with the previous kernel's tail

    const int m_tiles     = p.tiles_x * p.tiles_y * p.tiles_n;
    const int total_tiles = m_tiles * p.tiles_oc;
    const int num_kb      = p.ksize * p.ksize * p.cblocks;
    const int total_work  = SK ? p.sk_dp + 4 * p.sk_ctas : total_tiles * p.ksplit; // one past the last work id
    auto next_work = [&](int work) { return SK ? sk_next_work(p, work, (int) blockIdx.x, (int) gridDim.x, num_kb, total_work) : work + (int) gridDim.x; };
    const int first_work = SK ? sk_first_work(p, (int) blockIdx.x, total_work) : (int) blockIdx.x;
    EpiArgs e;
    e.o_hi64 = &tmO_hi64, e.o_lo64 = &tmO_lo64, e.o_hiT = &tmO_hiT, e.o_loT = &tmO_loT;
    e.r_hi64 = &tmR_hi64, e.r_lo64 = &tmR_lo64, e.r_hiT = &tmR_hiT, e.r_loT = &tmR_loT;
    e.bias = p.bias, e.OC = p.OC, e.act = p.act, e.has_res = p.has_res, e.rows_box = p.rows_used, e.alpha = p.alpha;
    e.has_lo = p.has_lo, e.stg = stg, e.stg_ready = stg_ready, e.stg_full = stg_full;

    if (wg == 0) {
        regs_dealloc_40(); // the consumers' two accumulator sets need the registers
        if (warp == 1) {
            // ===================== epilogue store thread =====================
            if (lane != 0) return;
            uint32_t full_phase = 0, dumped_phase = 0;
            for (int work = first_work; work < total_work; work = next_work(work)) {
                const WorkItem wi = decode_work<SK>(p, work, total_tiles, num_kb);
                if (wi.pieces > 1) {
                    // every consumer thread has dumped its part of the fp32 partial tile: count this piece's arrival. The last of
                    // the tile's pieces to arrive sums them (consumers, in piece order) and runs the epilogue; the others skip it.
                    mbar_wait(dumped_bar, dumped_phase);
                    dumped_phase ^= 1u;
                    __threadfence();
                    const int old  = atomicAdd(p.counters + wi.slot, 1);
                    const int last = old == wi.pieces - 1;
                    if (last) p.counters[wi.slot] = 0; // every piece has arrived: leave the counter ready for the next launch
                    asm volatile("st.shared.b32 [%0], %1;" ::"r"(last_flag), "r"(last) : "memory");
                    mbar_arrive(verdict_bar);
                    if (!last) continue;
                }
                const int m_idx = wi.tile % m_tiles, oc_idx = wi.tile / m_tiles;
                const int bx = m_idx % p.tiles_x, by = (m_idx / p.tiles_x) % p.tiles_y, bn = m_idx / (p.tiles_x * p.tiles_y);
                epilogue_store_tile<NB>(e, oc_idx * NB, bx * p.tw, by * p.th, bn * p.tn, full_phase);
            }
            epilogue_drain();
            return;
        }
        if (warp != 0) return;
        // ===================== TMA producer (one thread) =====================
        const uint32_t tx_bytes = (uint32_t) G::A_PLANES * (uint32_t) p.rows_used * 128u + (uint32_t) G::B_PLANES * (uint32_t) G::B_BYTES;
        const int ks = p.ksize, cbs = p.cblocks, icp = p.ICp;
        int stage = 0;
        uint32_t phase = 0;
        for (int work = first_work; work < total_work; work = next_work(work)) {
            const WorkItem wi = decode_work<SK>(p, work, total_tiles, num_kb);
            const int m_idx = wi.tile % m_tiles, oc_idx = wi.tile / m_tiles;
            const int bx = m_idx % p.tiles_x, by = (m_idx / p.tiles_x) % p.tiles_y, bn = m_idx / (p.tiles_x * p.tiles_y);
            const int ix0 = bx * p.tw * p.stride - p.pad_x, iy0 = by * p.th * p.stride - p.pad_y, n0 = bn * p.tn;
            const int oc0 = oc_idx * NB;
            // K block kb = (ky * ks + kx) * cbs + cb; the counters are decoded once per work item and then stepped
            int cb = wi.kb0 % cbs, tap0 = wi.kb0 / cbs;
            int kx = tap0 % ks, ky = tap0 / ks;
            int wk = tap0 * icp; // K coordinate into the packed weights = tap * ICp + cb * 64
            for (int kb = wi.kb0; kb < wi.kb1; ++kb) {
                mbar_wait(empty_bar(stage), phase ^ 1u);
                if (elect_one()) {
                    const uint32_t sA = smem_base + stage * G::STAGE_BYTES, sB = sA + G::A_PLANES * UM_A_BYTES, fb = full_bar(stage);
                    mbar_expect_tx(fb, tx_bytes);
                    tma_load_4d(sA, &tmA_hi, fb, cb * UM_BLOCK_K, ix0 + kx, iy0 + ky, n0);
                    if (TERMS >= 2) tma_load_4d(sA + UM_A_BYTES, &tmA_lo, fb, cb * UM_BLOCK_K, ix0 + kx, iy0 + ky, n0);
                    tma_load_2d(sB, &tmB_hi, fb, wk + cb * UM_BLOCK_K, oc0);
                    if (TERMS == 3) tma_load_2d(sB + G::B_BYTES, &tmB_lo, fb, wk + cb * UM_BLOCK_K, oc0);
                }
                __syncwarp();
                if (++stage == STAGES) stage = 0, phase ^= 1u;
                if (++cb == cbs) {
                    cb = 0, wk += icp;
                    if (++kx == ks) kx = 0, ++ky;
                }
            }
        }
        return;
    }

    // ===================== consumers: wgmma main loop + epilogue =====================
    regs_alloc_232();
    const int cw  = wg - 1;                                // consumer warpgroup: tile rows [64 cw, 64 cw + 64)
    const int wq  = warp & 3;                              // warp within the warpgroup
    const int row0 = 64 * cw + 16 * wq + (lane >> 2);      // tile row of d[0]; d[2] is row0 + 8
    const int q    = lane & 3;
    uint32_t ready_phase = 0, verdict_phase = 0;
    int stage = 0;
    uint32_t phase = 0;
    float acc[NB / 2], blk[NB / 2];
    // The two warpgroups take turns issuing K blocks (1: block k, 2: block k, 1: block k + 1, ...), each waiting for its turn on its
    // own named barrier and passing the turn on once its block's wgmmas are queued. So while one warpgroup drains its block
    // (wait_group 0, promotion, stage release) or runs its epilogue, the other one's wgmmas keep the tensor cores busy. The order is
    // seeded once and runs on across tiles and work items: both warpgroups walk the same K blocks.
    if (cw == 1) named_bar_arrive(UM_TURN_BAR, UM_EPI_THREADS);
    for (int work = first_work; work < total_work; work = next_work(work)) {
        const WorkItem wi = decode_work<SK>(p, work, total_tiles, num_kb);
#pragma unroll
        for (int i = 0; i < NB / 2; ++i) acc[i] = 0.0f;
        for (int kb = wi.kb0; kb < wi.kb1; ++kb) {
            mbar_wait(full_bar(stage), phase); // TMA bytes have landed
            const uint32_t sA = smem_base + stage * G::STAGE_BYTES, sB = sA + G::A_PLANES * UM_A_BYTES;
            const uint64_t a_hi = gmma_desc_sw128(sA + cw * 64 * 128), a_lo = gmma_desc_sw128(sA + UM_A_BYTES + cw * 64 * 128);
            const uint64_t b_hi = gmma_desc_sw128(sB), b_lo = gmma_desc_sw128(sB + G::B_BYTES);
            named_bar_sync(UM_TURN_BAR + cw, UM_EPI_THREADS); // my turn
            wg_fence();
#pragma unroll
            for (int k = 0; k < UM_BLOCK_K / 16; ++k) {
                Wgmma<NB>::mma(blk, a_hi + 2u * k, b_hi + 2u * k, k > 0 ? 1u : 0u);
                if (TERMS == 3) Wgmma<NB>::mma(blk, a_hi + 2u * k, b_lo + 2u * k, 1u);
                if (TERMS >= 2) Wgmma<NB>::mma(blk, a_lo + 2u * k, b_hi + 2u * k, 1u);
            }
            wg_commit();
            named_bar_arrive(UM_TURN_BAR + (cw ^ 1), UM_EPI_THREADS); // your turn
            wg_wait<0>(); // this K block's wgmmas have retired: its stage goes back to the producer
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(stage));
            acc_promote(acc, blk);
            if (++stage == STAGES) stage = 0, phase ^= 1u;
        }
        if (wi.pieces > 1) {
            // fp32 partial tile [row][NB]; the last of the tile's pieces to arrive sums them in piece order (deterministic). The store
            // thread counts the arrival once all 256 consumer threads have dumped theirs, and posts the verdict in last_flag.
            float* tile_parts = p.partials + (size_t) wi.slot * (SK ? 4 : p.ksplit) * (UM_BLOCK_M * NB);
            float* mine       = tile_parts + (size_t) wi.piece * (UM_BLOCK_M * NB);
#pragma unroll
            for (int j = 0; j < NB / 8; ++j)
#pragma unroll
                for (int r = 0; r < 2; ++r)
                    __stcg(reinterpret_cast<float2*>(mine + (size_t) (row0 + 8 * r) * NB + 8 * j + 2 * q), make_float2(acc[4 * j + 2 * r], acc[4 * j + 2 * r + 1]));
            __threadfence(); // partial tile visible device-wide before the arrival is counted
            mbar_arrive(dumped_bar);
            mbar_wait(verdict_bar, verdict_phase);
            verdict_phase ^= 1u;
            int last;
            asm volatile("ld.shared.b32 %0, [%1];" : "=r"(last) : "r"(last_flag) : "memory");
            if (!last) continue;
            __threadfence();
#pragma unroll
            for (int j = 0; j < NB / 8; ++j)
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const float* src = tile_parts + (size_t) (row0 + 8 * r) * NB + 8 * j + 2 * q;
                    float2 s = __ldcg(reinterpret_cast<const float2*>(src));
                    for (int sp = 1; sp < wi.pieces; ++sp) {
                        const float2 t = __ldcg(reinterpret_cast<const float2*>(src + (size_t) sp * (UM_BLOCK_M * NB)));
                        s.x += t.x, s.y += t.y;
                    }
                    acc[4 * j + 2 * r] = s.x, acc[4 * j + 2 * r + 1] = s.y;
                }
        }
        epilogue_tile<NB>(e, acc, (wi.tile / m_tiles) * NB, row0, q, ready_phase);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Small-input-channel convolution (IC <= 8: the 7x7 / 3x3 RGB stems, ESPCN's 1-channel 5x5) on the same tensor cores,
// with a ZERO-COPY sliding-window A operand.
//
// With C padded to 8 fp16 one pixel is ONE 16-byte vector per plane = exactly one K "core matrix" column of a wgmma K-major
// operand. In the un-swizzled canonical layout row m / chunk c of A is read from
//        start + (m/8)*SBO + (m%8)*16 B + c*LBO,
// and nothing stops LBO from being 16 B: chunk c of row m is then simply pixel m + c of a dense pixel row in shared
// memory - the convolution's sliding window, expressed in the descriptor.
// So for every filter row ky the producer TMA-loads ONE dense row segment per column parity (for stride 2 the even and
// odd input columns are de-interleaved by the tensor map's 32-byte pixel stride; out-of-image pixels are zero-filled =
// constant padding) and the consumers issue one K=16 step per pair of taps: no im2col, no copies.
// L2 -> SM traffic per 128-pixel tile: kh * s * ~136 * 16 B * 2 planes (61 KB for the 7x7 stem) instead of 224 KB of
// gathered 16-byte requests. The weight panel [kh][n_blk][64] (hi + lo, K columns in RowPlan order) is loaded once per
// persistent CTA and stays resident. Tiles = up to 128 consecutive output pixels of one output row.
//
// FEED mode (stride 2, <= 4 input channels = the RGB stems): the input kernels also write a compact copy of the image with
// FOUR channels per pixel and zero margins (snnb_tensor::feed_hi). With 8-byte pixels one 16-byte K chunk is a PAIR of adjacent
// pixels, and for stride 2 the window of output pixel m starts at pixel 2 m = 16 m bytes: the plain dense row is already the
// canonical operand (row pitch 16 B, LBO 16 B) - no parity de-interleave, half the K (7 taps x 4 channels + 1 pad tap = 32 instead of
// 64), one contiguous bulk copy per plane and filter row, real zeros instead of out-of-bounds fill (FeedPlan, snnb_internal.h).
// ---------------------------------------------------------------------------------------------------------------
constexpr int RW_THREADS       = UM_THREADS;
constexpr int RW_SMEM_BYTES    = UM_SMEM_LIMIT;                // everything: resident weight panels | epilogue staging | A ring | barriers

struct RowWinParams {
    const float* bias;
    int N, OH, OW, OC, OCp, n_blk;
    int kh, stride, pad_y;
    int tiles_x;
    int parities, dmin[2];
    int ksteps, panels, ks_parity[8], ks_erel[8]; // panels = ceil(ksteps / 4) weight panels of 64 K columns per filter row
    int act;
    float alpha;
    // FEED mode (stride 2, <= 4 input channels; FeedPlan in snnb_internal.h): the A rows come from the input tensor's compact
    // 4-channel copy, one contiguous segment per plane and filter row (a plain bulk copy, the margins are real zeros)
    const __half* feed_hi;
    const __half* feed_lo;
    int feed_h, feed_w, feed_py;
    uint32_t feed_seg_bytes; // 0 = not in feed mode
    // shared-memory carve-up (ConvPlan): the weight panels take b_bytes (multiple of 1024), the ring gets `stages` stages of
    // stage_bytes = planes x parities x RW_ARR_BYTES; the lo plane's arrays follow the hi plane's at lo_off. The ring is as deep as
    // shared memory allows: a stage is only ~2-9 KB and holds little work, so the producer has to run far ahead.
    int stages;
    uint32_t stage_bytes, lo_off, b_bytes;
    // FEED mode: a stage holds `rows_per_stage` filter rows (row_bytes each: hi segment, lo segment), released together
    int rows_per_stage;
    uint32_t row_bytes;
    int feed_prows; // feed mode: 128-byte weight rows per output channel = ceil(kh / FeedPlan::rows_per_panel)
};

// FKS > 0: FEED mode with FKS K steps per filter row (see RowWinParams::feed_hi). NB: n_blk (output channels, 32 or 64).
template <int TERMS, int FKS, int NB>
__global__ void __launch_bounds__(RW_THREADS, 1)
conv_rowwin_kernel(const __grid_constant__ CUtensorMap tmA_hi0, const __grid_constant__ CUtensorMap tmA_hi1, const __grid_constant__ CUtensorMap tmA_lo0,
                   const __grid_constant__ CUtensorMap tmA_lo1, const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
                   const __grid_constant__ CUtensorMap tmO_hi, const __grid_constant__ CUtensorMap tmO_lo, const RowWinParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t sB = smem_base; // weight panel: per (filter row, panel), [NB rows of B_hi ; NB rows of B_lo] x 128 B
    const uint32_t stg      = smem_base + p.b_bytes; // epilogue staging (1024-aligned)
    const uint32_t sA0      = stg + (uint32_t) UM_STG_BYTES;
    const uint32_t bar_base = sA0 + (uint32_t) p.stages * p.stage_bytes;
    const int RW_STAGES     = p.stages;
    auto full_bar       = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar      = [&](int s) { return bar_base + 8u * (RW_MAX_STAGES + s); };
    const uint32_t b_bar = bar_base + 8u * (2 * RW_MAX_STAGES);
    const uint32_t stg_ready = bar_base + 8u * (2 * RW_MAX_STAGES + 1), stg_full = bar_base + 8u * (2 * RW_MAX_STAGES + 2);
    static_assert(8 * (2 * RW_MAX_STAGES + 3) <= RW_BAR_BYTES, "barrier area");

    const int wg = threadIdx.x >> 7, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    pdl_trigger();
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA_hi0);
        tma_prefetch_desc(&tmA_lo0);
        tma_prefetch_desc(&tmB_hi);
        tma_prefetch_desc(&tmB_lo);
        for (int s = 0; s < RW_STAGES; ++s) {
            mbar_init(full_bar(s), 1);
            mbar_init(empty_bar(s), UM_EPI_THREADS / 32);
        }
        mbar_init(b_bar, 1);
        mbar_init(stg_ready, 1);
        mbar_init(stg_full, UM_EPI_THREADS);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();

    const int total_tiles = p.N * p.OH * p.tiles_x;
    constexpr uint32_t B_PLANE = (uint32_t) NB * 128u; // one weight plane of a panel
    EpiArgs e;
    // a 64-channel slab uses the swizzled map, a narrower one the dense map: the host encodes the right one into both slots
    e.o_hi64 = &tmO_hi, e.o_lo64 = &tmO_lo, e.o_hiT = &tmO_hi, e.o_loT = &tmO_lo;
    e.r_hi64 = e.r_lo64 = e.r_hiT = e.r_loT = &tmO_hi;
    e.bias = p.bias, e.OC = p.OC, e.act = p.act, e.has_res = 0, e.rows_box = UM_BLOCK_M, e.alpha = p.alpha;
    e.has_lo = TERMS >= 2, e.stg = stg, e.stg_ready = stg_ready, e.stg_full = stg_full;

    if (wg == 0) {
        regs_dealloc_40();
        if (warp == 1) {
            // epilogue store thread (see epilogue_store_tile)
            if (elect_one()) {
                uint32_t full_phase = 0;
                for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                    const int xt = tile % p.tiles_x, oy = (tile / p.tiles_x) % p.OH, n = tile / (p.tiles_x * p.OH);
                    epilogue_store_tile<NB>(e, 0, xt * UM_BLOCK_M, oy, n, full_phase);
                }
                epilogue_drain();
            }
            return;
        }
        if (warp != 0) return;
        // weight panels: once per CTA, [filter row][panel][plane] (feed mode: several filter rows share one 128-byte weight row)
        if (elect_one()) {
            const int vrows = FKS > 0 ? p.feed_prows : p.kh * p.panels;
            mbar_expect_tx(b_bar, (TERMS == 3 ? 2u : 1u) * (uint32_t) vrows * B_PLANE);
            for (int v = 0; v < vrows; ++v) {
                if (TERMS == 3) {
                    tma_load_3d(sB + (2 * v) * B_PLANE, &tmB_hi, b_bar, 0, 0, v);
                    tma_load_3d(sB + (2 * v + 1) * B_PLANE, &tmB_lo, b_bar, 0, 0, v);
                } else {
                    tma_load_3d(sB + v * B_PLANE, &tmB_hi, b_bar, 0, 0, v); // one plane
                }
            }
        }
        __syncwarp();
        // activation row segments
        int stage = 0;
        uint32_t phase = 0;
        const uint32_t tx_bytes = (TERMS == 1 ? 1u : 2u) * (p.feed_seg_bytes ? p.feed_seg_bytes : (uint32_t) p.parities * RW_ARR_BYTES);
        if constexpr (FKS > 0) {
            // one contiguous segment per plane and filter row; running pointers, no per-stage address arithmetic
            const uint32_t seg  = p.feed_seg_bytes;
            const size_t pitch  = (size_t) p.feed_w * 4; // fp16 elements per feed row
            const int per_image = p.OH * p.tiles_x;
            int rem = (int) blockIdx.x % per_image, n = (int) blockIdx.x / per_image;
            uint32_t sA = sA0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int oy = p.tiles_x == 1 ? rem : rem / p.tiles_x, xt = p.tiles_x == 1 ? 0 : rem % p.tiles_x;
                const size_t off = (((size_t) n * p.feed_h + (oy * 2 - p.pad_y + p.feed_py)) * p.feed_w + 2 * xt * UM_BLOCK_M) * 4;
                const __half* src_hi = p.feed_hi + off;
                const __half* src_lo = p.feed_lo + off;
                for (int ky0 = 0; ky0 < p.kh; ky0 += p.rows_per_stage) {
                    const int rows = min(p.rows_per_stage, p.kh - ky0); // this stage's group of filter rows
                    mbar_wait(empty_bar(stage), phase ^ 1u);
                    if (elect_one()) {
                        mbar_expect_tx(full_bar(stage), tx_bytes * (uint32_t) rows);
                        const __half* sh = src_hi;
                        const __half* sl = src_lo;
                        uint32_t dst     = sA;
                        for (int r = 0; r < rows; ++r, dst += p.row_bytes, sh += pitch, sl += pitch) {
                            bulk_load_1d(dst, sh, seg, full_bar(stage));
                            if (TERMS >= 2) bulk_load_1d(dst + RW_ARR_BYTES, sl, seg, full_bar(stage));
                        }
                    }
                    __syncwarp();
                    src_hi += pitch * rows, src_lo += pitch * rows;
                    sA += p.stage_bytes;
                    if (++stage == RW_STAGES) stage = 0, phase ^= 1u, sA = sA0;
                }
                rem += (int) gridDim.x;
                while (rem >= per_image) rem -= per_image, ++n;
            }
        } else {
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int xt = tile % p.tiles_x, oy = (tile / p.tiles_x) % p.OH, n = tile / (p.tiles_x * p.OH);
                const int ox0 = xt * UM_BLOCK_M;
                for (int ky = 0; ky < p.kh; ++ky) {
                    const int iy = oy * p.stride - p.pad_y + ky; // out of range -> the whole row is zero-filled
                    mbar_wait(empty_bar(stage), phase ^ 1u);
                    if (elect_one()) {
                        const uint32_t sA = sA0 + stage * p.stage_bytes;
                        mbar_expect_tx(full_bar(stage), tx_bytes);
                        tma_load_4d(sA, &tmA_hi0, full_bar(stage), 0, ox0 + p.dmin[0], iy, n);
                        if (TERMS >= 2) tma_load_4d(sA + p.lo_off, &tmA_lo0, full_bar(stage), 0, ox0 + p.dmin[0], iy, n);
                        if (p.parities == 2) {
                            tma_load_4d(sA + RW_ARR_BYTES, &tmA_hi1, full_bar(stage), 0, ox0 + p.dmin[1], iy, n);
                            if (TERMS >= 2) tma_load_4d(sA + p.lo_off + RW_ARR_BYTES, &tmA_lo1, full_bar(stage), 0, ox0 + p.dmin[1], iy, n);
                        }
                    }
                    __syncwarp();
                    if (++stage == RW_STAGES) stage = 0, phase ^= 1u;
                }
            }
        }
        return;
    }

    // ===================== consumers =====================
    regs_alloc_232();
    const int cw   = wg - 1;
    const int row0 = 64 * cw + 16 * (warp & 3) + (lane >> 2);
    const int q    = lane & 3;
    uint32_t ready_phase = 0;
    mbar_wait(b_bar, 0);
    // window descriptor of this warpgroup's 64 rows (64 pixels x 16 B further into the row segment)
    const uint64_t wdesc0 = gmma_desc_window(sA0 + (uint32_t) cw * 64u * 16u), bdesc0 = gmma_desc_sw128(sB);
    const uint32_t b_panel = (uint32_t) ((TERMS == 3 ? 2 : 1) * NB * 128) >> 4; // one [B_hi ; B_lo] (or single-plane) panel (64 K columns)
    const uint32_t b_lo16  = B_PLANE >> 4;
    const uint64_t lo16    = (uint64_t) (p.lo_off >> 4);
    int stage = 0;
    uint32_t phase = 0;
    float acc[NB / 2], blk[NB / 2];
    // one K=16 step of the product into the stage's fresh accumulator: A window at `a` (hi plane; lo plane at + alo), weights at `b`
    auto kstep = [&](uint64_t a, uint64_t alo, uint64_t b, uint32_t accumulate) {
        Wgmma<NB>::mma(blk, a, b, accumulate);
        if (TERMS == 3) Wgmma<NB>::mma(blk, a, b + b_lo16, 1u);
        if (TERMS >= 2) Wgmma<NB>::mma(blk, a + alo, b, 1u);
    };
    // the stage's wgmmas have retired: hand the stage back to the producer, add the stage's sum to the tile's
    auto finish_stage = [&]() {
        wg_commit();
        wg_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(stage));
        acc_promote(acc, blk);
        if (++stage == RW_STAGES) stage = 0, phase ^= 1u;
    };
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
#pragma unroll
        for (int i = 0; i < NB / 2; ++i) acc[i] = 0.0f;
        if constexpr (FKS > 0) {
            // K step q of a filter row = window start + 2 q pixel pairs (32 B), weight columns 16 q ..
            constexpr int RPP     = FKS == 1 ? 4 : (FKS == 2 ? 2 : 1); // FeedPlan::rows_per_panel
            const uint32_t row16  = p.row_bytes >> 4;
            uint64_t b_cat        = bdesc0;
            int b_sub             = 0;
            for (int ky0 = 0; ky0 < p.kh; ky0 += p.rows_per_stage) {
                const int rows = min(p.rows_per_stage, p.kh - ky0);
                mbar_wait(full_bar(stage), phase);
                uint64_t a_row = wdesc0 + (uint64_t) ((uint32_t) stage * (p.stage_bytes >> 4));
                wg_fence();
                for (int r = 0; r < rows; ++r, a_row += row16) {
                    // weights of this filter row: the next K-column group of the same 128-byte rows, or the next panel
                    const uint64_t b_now = b_cat;
                    if (++b_sub == RPP) b_sub = 0, b_cat += b_panel - (RPP - 1) * (8 / RPP);
                    else b_cat += 8 / RPP;
#pragma unroll
                    for (int k = 0; k < FKS; ++k) kstep(a_row + 2u * k, (uint64_t) (RW_ARR_BYTES >> 4), b_now + 2u * k, (r > 0 || k > 0) ? 1u : 0u);
                }
                finish_stage();
            }
        } else {
            const uint32_t b_ky = b_panel * (uint32_t) p.panels; // one filter row
            for (int ky = 0; ky < p.kh; ++ky) {
                mbar_wait(full_bar(stage), phase);
                const uint64_t a0 = wdesc0 + (uint64_t) ((uint32_t) stage * (p.stage_bytes >> 4));
                const uint64_t bk = bdesc0 + (uint64_t) ((uint32_t) ky * b_ky);
                wg_fence();
#pragma unroll
                for (int k = 0; k < 8; ++k) { // K step k: parity ks_parity[k], window offset ks_erel[k]; weight panel k / 4, columns 16 (k % 4) ..
                    if (k < p.ksteps) {
                        const uint32_t koff = ((uint32_t) p.ks_parity[k] * RW_ARR_BYTES + (uint32_t) p.ks_erel[k] * 16u) >> 4;
                        kstep(a0 + koff, lo16, bk + (uint64_t) ((k >> 2) * b_panel + 2u * (k & 3)), k > 0 ? 1u : 0u);
                    }
                }
                finish_stage();
            }
        }
        epilogue_tile<NB>(e, acc, 0, row0, q, ready_phase);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Host side: tensor maps and launch of what the convolution planner decided (conv_plan.cpp, ConvPlan)
// ---------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode(snnb_context* ctx) {
    if (!ctx->tmap_encode_fn) {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess) return nullptr;
        ctx->tmap_encode_fn = fn;
    }
    return reinterpret_cast<EncodeTiledFn>(ctx->tmap_encode_fn);
}

// Tensor maps of an NHWC split-fp16 tensor for the epilogue's TMA stores / residual loads: box = (width channels, tw, th, tn).
static int encode_nhwc_box_maps(EncodeTiledFn encode, const snnb_tensor* t, int width, int tw, int th, int tn, bool swizzle128, CUtensorMap (&maps)[2]) {
    const cuuint64_t dims[4]    = {(cuuint64_t) t->cp, (cuuint64_t) t->w, (cuuint64_t) t->h, (cuuint64_t) t->n};
    const cuuint64_t strides[3] = {(cuuint64_t) t->cp * 2, (cuuint64_t) t->w * t->cp * 2, (cuuint64_t) t->h * t->w * t->cp * 2};
    const cuuint32_t box[4]     = {(cuuint32_t) width, (cuuint32_t) tw, (cuuint32_t) th, (cuuint32_t) tn};
    const cuuint32_t estr[4]    = {1, 1, 1, 1};
    __half* planes[2]    = {t->hi, t->lo ? t->lo : t->hi}; // fp16 storage mode: the lo map is encoded but never used
    for (int i = 0; i < 2; ++i) {
        CUresult r = encode(&maps[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, planes[i], dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        SNNB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(out/residual) failed: %d (cp %d w %d h %d n %d box %d %d %d %d)", (int) r, t->cp, t->w, t->h, t->n,
                     width, tw, th, tn);
    }
    return 0;
}

// fp32 partial tiles + arrival counters of split-K launches. Grow-only, old blocks stay alive until the context dies:
// captured CUDA graphs keep the pointers they were recorded with.
static int ensure_splitk_scratch(snnb_context* ctx, size_t partial_bytes, size_t n_counters) {
    if (partial_bytes > ctx->splitk_bytes) {
        void* pnew = nullptr;
        SNNB_CUDA_OK(cudaMalloc(&pnew, partial_bytes));
        ctx->scratch_blocks.push_back(pnew);
        ctx->splitk_partials = static_cast<float*>(pnew), ctx->splitk_bytes = partial_bytes;
    }
    if (n_counters > ctx->splitk_counter_n) {
        void* pnew = nullptr;
        SNNB_CUDA_OK(cudaMalloc(&pnew, n_counters * sizeof(int)));
        SNNB_CUDA_OK(cudaMemset(pnew, 0, n_counters * sizeof(int)));
        ctx->scratch_blocks.push_back(pnew);
        ctx->splitk_counters = static_cast<int*>(pnew), ctx->splitk_counter_n = n_counters;
    }
    return 0;
}

// Bits of snnb_context::func_attr_mask (cudaFuncSetAttribute applies per device): one per kernel instantiation
enum { ATTR_UMMA0 = 0, ATTR_ROWWIN0 = 18, ATTR_DW1 = 48, ATTR_DW2 = 49 };
static int ensure_smem_attr(snnb_context* ctx, const void* kernel, int bit, int bytes) {
    const uint64_t m = 1ull << bit;
    if (!(ctx->func_attr_mask & m)) {
        SNNB_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        ctx->func_attr_mask |= m;
    }
    return 0;
}

typedef void (*UmmaKernel)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap,
                           const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const UmmaParams);
struct UmmaChoice {
    UmmaKernel kernel;
    int smem, bit;
};
template <int TERMS, int NB> static UmmaChoice umma_choice_nb(bool sk, int nbi) {
    return {sk ? conv_umma_kernel<TERMS, NB, true> : conv_umma_kernel<TERMS, NB, false>, UmGeom<TERMS, NB>::SMEM_BYTES, ATTR_UMMA0 + ((TERMS - 1) * 3 + nbi) * 2 + (sk ? 1 : 0)};
}
template <int TERMS> static UmmaChoice umma_choice_t(int nb, bool sk) {
    return nb == 32 ? umma_choice_nb<TERMS, 32>(sk, 0) : (nb == 64 ? umma_choice_nb<TERMS, 64>(sk, 1) : umma_choice_nb<TERMS, 128>(sk, 2));
}
static UmmaChoice umma_choice(int terms, int nb, bool sk) { return terms == 3 ? umma_choice_t<3>(nb, sk) : (terms == 2 ? umma_choice_t<2>(nb, sk) : umma_choice_t<1>(nb, sk)); }

typedef void (*RowWinKernel)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap, const CUtensorMap,
                             const CUtensorMap, const RowWinParams);
template <int TERMS, int NB> static RowWinKernel rowwin_kernel_fks(int fks) {
    switch (fks) {
    case 1: return conv_rowwin_kernel<TERMS, 1, NB>;
    case 2: return conv_rowwin_kernel<TERMS, 2, NB>;
    case 3: return conv_rowwin_kernel<TERMS, 3, NB>;
    default: return conv_rowwin_kernel<TERMS, 0, NB>;
    }
}
template <int TERMS> static RowWinKernel rowwin_kernel_t(int fks, int nb) { return nb == 32 ? rowwin_kernel_fks<TERMS, 32>(fks) : rowwin_kernel_fks<TERMS, 64>(fks); }
static RowWinKernel rowwin_kernel_of(int terms, int fks, int nb) {
    return terms == 3 ? rowwin_kernel_t<3>(fks, nb) : (terms == 2 ? rowwin_kernel_t<2>(fks, nb) : rowwin_kernel_t<1>(fks, nb));
}

int launch_conv2d_rowwin(snnb_context* ctx, const ConvArgs& a, const ConvPlan& plan) {
    EncodeTiledFn encode = get_encode(ctx);
    SNNB_REQUIRE(encode, "launch_conv2d_rowwin: cuTensorMapEncodeTiled is unavailable in this driver");
    const snnb_tensor* in = a.in;
    snnb_tensor* out      = a.out;
    const bool feed       = plan.path == CONV_ROWWIN_FEED;
    SNNB_REQUIRE(plan.path == CONV_ROWWIN || feed, "launch_conv2d_rowwin: the plan is not a row-window launch");
    SNNB_REQUIRE(a.w->w_row_hi && a.w->w_row_lo && a.w->row_stride == a.stride && a.w->row_pad == a.pad_x,
                 "launch_conv2d_rowwin: the weights carry no row-window operand for stride %d, pad %d", a.stride, a.pad_x);
    SNNB_REQUIRE(feed || !in->feed_only, "launch_conv2d_rowwin: the input tensor only exists as a stem feed, which this launch cannot read");
    SNNB_REQUIRE(!feed || (a.w->w_feed_hi && a.w->w_feed_lo && a.w->feed_pad == a.pad_x), "launch_conv2d_rowwin: the weights carry no feed operand for pad %d", a.pad_x);
    SNNB_REQUIRE(!feed || (in->feed_hi && in->feed_h == plan.feed_h && in->feed_w == plan.feed_w && in->feed_py == plan.feed_py && in->feed_px == plan.feed_px),
                 "launch_conv2d_rowwin: the input tensor does not carry the planned feed copy");
    SNNB_REQUIRE(out->n == plan.n && (plan.terms == 1 || (in->lo && out->lo)),
                 "launch_conv2d_rowwin: the tensors do not match the plan (batch %d, %d-term product)", plan.n, plan.terms);
    const RowPlan& rp = plan.rp;
    ctx->last_kernel  = feed ? "conv_rowwin_kernel<feed>" : "conv_rowwin_kernel";
    SNNB_REQUIRE(plan.stages >= 2, "launch_conv2d_rowwin: weight panels of %u bytes leave no room for the activation ring", plan.b_bytes);
    RowWinParams p;
    p.bias = a.w->bias;
    p.N = out->n, p.OH = out->h, p.OW = out->w, p.OC = out->c, p.OCp = out->cp;
    p.n_blk = plan.n_blk;
    p.kh = a.k, p.stride = a.stride, p.pad_y = a.pad_y;
    p.tiles_x  = plan.tiles_x;
    p.parities = rp.parities, p.dmin[0] = rp.dmin[0], p.dmin[1] = rp.dmin[1];
    p.ksteps   = rp.ksteps, p.panels = plan.panels;
    std::copy(rp.ks_parity, rp.ks_parity + 8, p.ks_parity);
    std::copy(rp.ks_erel, rp.ks_erel + 8, p.ks_erel);
    p.act = a.act, p.alpha = a.alpha;
    p.feed_hi = in->feed_hi, p.feed_lo = in->feed_lo, p.feed_h = in->feed_h, p.feed_w = in->feed_w, p.feed_py = in->feed_py;
    p.feed_seg_bytes = plan.feed_seg_bytes;
    p.lo_off         = plan.lo_off;
    p.row_bytes      = plan.row_bytes;
    p.rows_per_stage = plan.rows_per_stage;
    p.stage_bytes    = plan.stage_bytes;
    p.feed_prows     = feed ? plan.wrows : 0;
    p.b_bytes        = plan.b_bytes;
    p.stages         = plan.stages;

    // A: per plane and column parity a 4-D view (8 ch | de-interleaved pixel index | row | image) of the NHWC plane
    CUtensorMap tmA[4], tmB[2];
    for (int plane = 0; plane < 2; ++plane)
        for (int par = 0; par < 2; ++par) {
            const int pp = par < rp.parities ? par : 0; // unused maps alias parity 0 (kernel never issues them)
            __half* base = ((plane && in->lo) ? in->lo : in->hi) + (size_t) pp * 8; // half-precision storage mode: the lo maps are never issued
            const int wp        = (in->w - pp + a.stride - 1) / a.stride; // pixels of this parity per row
            const cuuint64_t dims[4]    = {8, (cuuint64_t) (wp > 0 ? wp : 1), (cuuint64_t) in->h, (cuuint64_t) in->n};
            const cuuint64_t strides[3] = {(cuuint64_t) a.stride * 16, (cuuint64_t) in->w * 16, (cuuint64_t) in->h * in->w * 16};
            const cuuint32_t box[4]     = {8, (cuuint32_t) RW_BOXW, 1, 1};
            const cuuint32_t estr[4]    = {1, 1, 1, 1};
            CUresult r = encode(&tmA[plane * 2 + par], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            SNNB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(A, rowwin) failed: %d", (int) r);
        }
    {
        // [weight row v][OCr][64 K columns]; a box of n_blk channel rows reads zeros past OCr
        const cuuint64_t dims[3]    = {64, (cuuint64_t) a.w->ocr, (cuuint64_t) plan.wrows};
        const cuuint64_t strides[2] = {128, (cuuint64_t) a.w->ocr * 128};
        const cuuint32_t box[3]     = {64, (cuuint32_t) p.n_blk, 1};
        const cuuint32_t estr[3]    = {1, 1, 1};
        void* planes[2] = {(void*) (feed ? a.w->w_feed_hi : a.w->w_row_hi), (void*) (feed ? a.w->w_feed_lo : a.w->w_row_lo)}; // 2-term: the hi plane alone = fp16_rn(w)
        for (int i = 0; i < 2; ++i) {
            CUresult r = encode(&tmB[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, planes[i], dims, strides, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            SNNB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(B, rowwin) failed: %d", (int) r);
        }
    }
    CUtensorMap tmO[2];
    if (encode_nhwc_box_maps(encode, out, p.n_blk, UM_BLOCK_M, 1, 1, p.n_blk == 64, tmO)) return 2;
    auto* kern           = rowwin_kernel_of(plan.terms, plan.fks, p.n_blk);
    const int variant[6] = {plan.path, plan.terms, p.n_blk, 1, 0, plan.fks};
    std::copy(variant, variant + 6, ctx->last_conv);
    if (ensure_smem_attr(ctx, (const void*) kern, ATTR_ROWWIN0 + ((plan.terms - 1) * 5 + plan.fks) * 2 + (p.n_blk == 64 ? 1 : 0), RW_SMEM_BYTES)) return 1;
    return launch_done(ctx, launch_k_pdl(kern, dim3(plan.grid), dim3(RW_THREADS), RW_SMEM_BYTES, ctx->stream, tmA[0], tmA[1], tmA[2], tmA[3], tmB[0], tmB[1], tmO[0], tmO[1], p), "conv_rowwin_kernel");
}

int launch_conv2d_umma(snnb_context* ctx, const ConvArgs& a, const ConvPlan& plan) {
    EncodeTiledFn encode = get_encode(ctx);
    SNNB_REQUIRE(encode, "launch_conv2d_umma: cuTensorMapEncodeTiled is unavailable in this driver");
    SNNB_REQUIRE(!a.in->feed_only, "launch_conv2d_umma: the input tensor only exists as a stem feed, which this launch cannot read");
    const snnb_tensor* in = a.in;
    snnb_tensor* out      = a.out;
    SNNB_REQUIRE(out->n == plan.n && (plan.terms == 1 || (in->lo && out->lo)),
                 "launch_conv2d_umma: the tensors do not match the plan (batch %d, %d-term product)", plan.n, plan.terms);
    UmmaParams p;
    p.has_res = a.residual != nullptr;
    p.bias    = a.w->bias;
    p.N = out->n, p.OH = out->h, p.OW = out->w, p.OC = out->c, p.OCp = out->cp;
    SNNB_REQUIRE(plan.tw > 0, "launch_conv2d_umma: no tile plan");
    p.tw = plan.tw, p.th = plan.th, p.tn = plan.tn, p.rows_used = plan.tw * plan.th * plan.tn;
    p.tiles_x = plan.tiles_x, p.tiles_y = plan.tiles_y, p.tiles_n = plan.tiles_n;
    p.ksize = a.k, p.stride = a.stride, p.pad_x = a.pad_x, p.pad_y = a.pad_y;
    p.cblocks = (in->c + UM_BLOCK_K - 1) / UM_BLOCK_K;
    p.has_lo  = out->lo != nullptr;
    SNNB_REQUIRE(plan.n_blk > 0, "launch_conv2d_umma: no output-channel plan");
    p.n_blk = plan.n_blk, p.tiles_oc = plan.tiles_oc, p.ksplit = plan.ksplit, p.kb_per_split = plan.kb_per_split;
    p.sk = plan.sk, p.sk_dp = plan.sk_dp, p.sk_ctas = plan.sk_ctas, p.sk_units = plan.sk_units;
    p.partials = nullptr, p.counters = nullptr;
    if (p.ksplit > 1 || p.sk) {
        // partial-tile slots: split-K [tile][split]; stream-K [tile past sk_dp][4 pieces]
        const size_t tiles = (size_t) plan.partial_tiles;
        cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
        SNNB_CUDA_OK(cudaStreamIsCapturing(ctx->stream, &cap));
        const size_t need = (size_t) plan.partial_slots * UM_BLOCK_M * p.n_blk * sizeof(float);
        SNNB_REQUIRE(cap == cudaStreamCaptureStatusNone || (need <= ctx->splitk_bytes && tiles <= ctx->splitk_counter_n),
                     "launch_conv2d_umma: split-K scratch must be allocated by an eager pass before graph capture");
        if (ensure_splitk_scratch(ctx, need, tiles)) return 1;
        p.partials = ctx->splitk_partials, p.counters = ctx->splitk_counters;
    }
    p.ICp     = round_up(in->c, 8);
    p.act = a.act, p.alpha = a.alpha;
    SNNB_REQUIRE(a.w->kp == a.k * a.k * p.ICp, "launch_conv2d_umma: packed weights do not match (kp %d vs %d)", a.w->kp, a.k * a.k * p.ICp);

    CUtensorMap tmA[2], tmB[2];
    {
        const cuuint64_t dims[4]    = {(cuuint64_t) in->c, (cuuint64_t) in->w, (cuuint64_t) in->h, (cuuint64_t) in->n};
        const cuuint64_t strides[3] = {(cuuint64_t) in->cp * 2, (cuuint64_t) in->w * in->cp * 2, (cuuint64_t) in->h * in->w * in->cp * 2};
        const cuuint32_t box[4]     = {(cuuint32_t) UM_BLOCK_K, (cuuint32_t) (p.tw * a.stride), (cuuint32_t) (p.th * a.stride), (cuuint32_t) p.tn};
        const cuuint32_t estr[4]    = {1, (cuuint32_t) a.stride, (cuuint32_t) a.stride, 1};
        __half* planes[2]    = {in->hi, in->lo ? in->lo : in->hi}; // fp16 storage mode: the lo map is never issued
        for (int i = 0; i < 2; ++i) {
            CUresult r = encode(&tmA[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, planes[i], dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            SNNB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(A) failed: %d (dims %d %d %d %d box %u %u %u %u)", (int) r, in->c, in->w, in->h, in->n, box[0],
                         box[1], box[2], box[3]);
        }
    }
    {
        const cuuint64_t dims[2]    = {(cuuint64_t) a.w->kp, (cuuint64_t) a.w->ocr};
        const cuuint64_t strides[1] = {(cuuint64_t) a.w->kp * 2};
        const cuuint32_t box[2]     = {(cuuint32_t) UM_BLOCK_K, (cuuint32_t) p.n_blk};
        const cuuint32_t estr[2]    = {1, 1};
        void* planes[2]             = {(void*) a.w->w_hi, (void*) a.w->w_lo}; // the 2-term product uses the hi plane alone: fp16_rn(w)
        for (int i = 0; i < 2; ++i) {
            CUresult r = encode(&tmB[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, planes[i], dims, strides, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            SNNB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(B) failed: %d (kp %d ocr %d n_blk %d)", (int) r, a.w->kp, a.w->ocr, p.n_blk);
        }
    }
    // epilogue maps: full 64-channel slabs (swizzled) and the narrow slab of a 32-channel tile (dense)
    CUtensorMap tmO64[2], tmOT[2], tmR64[2], tmRT[2];
    {
        const int wT = p.n_blk % 64;
        const snnb_tensor* res = a.residual ? a.residual : out;
        if (encode_nhwc_box_maps(encode, out, p.n_blk >= 64 ? 64 : wT, p.tw, p.th, p.tn, p.n_blk >= 64, tmO64)) return 2;
        if (encode_nhwc_box_maps(encode, out, wT ? wT : 64, p.tw, p.th, p.tn, wT == 0, tmOT)) return 2;
        if (encode_nhwc_box_maps(encode, res, p.n_blk >= 64 ? 64 : wT, p.tw, p.th, p.tn, p.n_blk >= 64, tmR64)) return 2;
        if (encode_nhwc_box_maps(encode, res, wT ? wT : 64, p.tw, p.th, p.tn, wT == 0, tmRT)) return 2;
    }
    const UmmaChoice kc = umma_choice(plan.terms, p.n_blk, p.sk != 0);
    if (ensure_smem_attr(ctx, (const void*) kc.kernel, kc.bit, kc.smem)) return 1;
    ctx->last_kernel = p.sk ? "conv_umma_kernel<stream-K>" : (p.ksplit > 1 ? "conv_umma_kernel<split-K>" : "conv_umma_kernel");
    const int variant[6] = {CONV_IGEMM, plan.terms, p.n_blk, p.ksplit, p.sk ? 1 : 0, 0};
    std::copy(variant, variant + 6, ctx->last_conv);
    return launch_done(ctx, launch_k_pdl(kc.kernel, dim3(plan.grid), dim3(UM_THREADS), kc.smem, ctx->stream, tmA[0], tmA[1], tmB[0], tmB[1], tmO64[0], tmO64[1], tmOT[0], tmOT[1],
                            tmR64[0], tmR64[1], tmRT[0], tmRT[1], p), "conv_umma_kernel");
}

// ---------------------------------------------------------------------------------------------------------------
// Depthwise 3x3 (stride 1 / 2), TMA-staged + register-tiled (shadertemplate_vk_depthwise.comp:64-139).
//
// HBM-bound work: every input byte should cross the memory system once. A persistent CTA walks tiles of
// TH x TW output pixels x 64 channels; for each tile ONE TMA box load per plane brings the (TH-1)*S+3 x (TW-1)*S+3
// input patch (128-byte pixel rows, no swizzle; out-of-image pixels and channels >= C are zero-filled = the zero padding)
// into a 3-deep shared-memory ring, so loads of the next tiles are in flight while this one is computed. A thread owns
// 8 channels (one 16-byte piece of the pixel row) and TXT consecutive output columns and streams the patch rows through
// registers (stride 1: 18 pixel loads for 4 outputs). A warp reads 4 pixel rows x 128 B per instruction: conflict-free.
// Outputs go straight to global memory: a warp writes 4 full 128-byte lines per plane.
// ---------------------------------------------------------------------------------------------------------------
constexpr int DW_THREADS = 256;
constexpr int DW_STAGES  = 2;
template <int S> struct DwTile {
    static constexpr int TW = S == 1 ? 16 : 8, TH = S == 1 ? 8 : 4; // output pixels per tile: 128 / 32
    static constexpr int TXT = S == 1 ? 4 : 1;                      // output columns per thread
    static constexpr int IW = (TW - 1) * S + 3, IH = (TH - 1) * S + 3;
    static constexpr int PLANE_BYTES = IW * IH * 128;
    static constexpr int STAGE_BYTES = 2 * PLANE_BYTES;
    static constexpr int SMEM_BYTES  = DW_STAGES * STAGE_BYTES + 128 /*alignment*/ + 64 /*barriers*/;
};
struct DwTmaParams {
    __half* out_hi;
    __half* out_lo;
    const float* w;    // [9][Cp]
    const float* bias; // [Cp + padding]
    int N, OH, OW, C, Cp;
    int pad_x, pad_y;
    int tiles_x, tiles_y, chunks;
    int act;
    float alpha;
};

template <int S>
__global__ void __launch_bounds__(DW_THREADS, 2) depthwise_tma_kernel(const __grid_constant__ CUtensorMap tmI_hi, const __grid_constant__ CUtensorMap tmI_lo, const DwTmaParams p) {
    using T = DwTile<S>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 127u) & ~127u;
    const uint32_t bar_base  = smem_base + DW_STAGES * T::STAGE_BYTES;
    const int tid = threadIdx.x, warp = tid >> 5;
    pdl_trigger();
    if (tid == 0) {
        tma_prefetch_desc(&tmI_hi);
        tma_prefetch_desc(&tmI_lo);
        for (int s = 0; s < DW_STAGES; ++s) mbar_init(bar_base + 8u * s, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();

    const int sp_tiles = p.N * p.tiles_y * p.tiles_x;
    const int total    = sp_tiles * p.chunks; // chunk is the slowest index: a CTA's consecutive tiles share its weights
    auto issue = [&](int tile, int stage) {   // one thread
        const int chunk = tile / sp_tiles, sp = tile - chunk * sp_tiles;
        const int tx = sp % p.tiles_x, ty = (sp / p.tiles_x) % p.tiles_y, n = sp / (p.tiles_x * p.tiles_y);
        const uint32_t dst = smem_base + stage * T::STAGE_BYTES, bar = bar_base + 8u * stage;
        mbar_expect_tx(bar, T::STAGE_BYTES);
        tma_load_4d(dst, &tmI_hi, bar, chunk * 64, tx * T::TW * S - p.pad_x, ty * T::TH * S - p.pad_y, n);
        tma_load_4d(dst + T::PLANE_BYTES, &tmI_lo, bar, chunk * 64, tx * T::TW * S - p.pad_x, ty * T::TH * S - p.pad_y, n);
    };
    if (tid == 0)
        for (int j = 0; j < DW_STAGES; ++j) {
            const int tile = blockIdx.x + j * gridDim.x;
            if (tile < total) issue(tile, j);
        }

    const int cg  = tid & 7, pt = tid >> 3;                                            // 16-byte channel piece, pixel-thread 0..31
    const int tyl = S == 1 ? (pt >> 2) : (pt >> 3), txl = S == 1 ? (pt & 3) * 4 : (pt & 7); // first output (row, col) in the tile
    const float slope   = (p.act == SNNB_ACT_RELU || p.act == SNNB_ACT_RELU6) ? 0.0f : (p.act == SNNB_ACT_LEAKY_RELU ? p.alpha : 1.0f);
    const float hi_clip = p.act == SNNB_ACT_RELU6 ? 6.0f : __int_as_float(0x7f800000);
    const bool fast_act = p.act == SNNB_ACT_NONE || p.act == SNNB_ACT_RELU || p.act == SNNB_ACT_RELU6 || p.act == SNNB_ACT_LEAKY_RELU;

    float wreg[9][8], breg[8];
    int cur_chunk = -1;
    int it = 0;
    for (int tile = blockIdx.x; tile < total; tile += gridDim.x, ++it) {
        const int stage = it % DW_STAGES;
        const int chunk = tile / sp_tiles, sp = tile - chunk * sp_tiles;
        const int tx = sp % p.tiles_x, ty = (sp / p.tiles_x) % p.tiles_y, n = sp / (p.tiles_x * p.tiles_y);
        const int c = chunk * 64 + cg * 8;
        if (chunk != cur_chunk) { // this thread's 8 channels of the folded weights and bias
            cur_chunk = chunk;
#pragma unroll
            for (int t = 0; t < 9; ++t) {
                float4 w0 = make_float4(0.f, 0.f, 0.f, 0.f), w1 = w0;
                if (c < p.Cp) {
                    w0 = __ldg(reinterpret_cast<const float4*>(p.w + (size_t) t * p.Cp + c));
                    w1 = __ldg(reinterpret_cast<const float4*>(p.w + (size_t) t * p.Cp + c) + 1);
                }
                wreg[t][0] = w0.x, wreg[t][1] = w0.y, wreg[t][2] = w0.z, wreg[t][3] = w0.w;
                wreg[t][4] = w1.x, wreg[t][5] = w1.y, wreg[t][6] = w1.z, wreg[t][7] = w1.w;
            }
            float4 b0 = make_float4(0.f, 0.f, 0.f, 0.f), b1 = b0;
            if (c < p.Cp) {
                b0 = __ldg(reinterpret_cast<const float4*>(p.bias + c));
                b1 = __ldg(reinterpret_cast<const float4*>(p.bias + c) + 1);
            }
            breg[0] = b0.x, breg[1] = b0.y, breg[2] = b0.z, breg[3] = b0.w, breg[4] = b1.x, breg[5] = b1.y, breg[6] = b1.z, breg[7] = b1.w;
        }
        mbar_wait(bar_base + 8u * stage, (uint32_t) (it / DW_STAGES) & 1u);
        const uint32_t src = smem_base + stage * T::STAGE_BYTES + (uint32_t) cg * 16u;

        float acc[T::TXT][8];
#pragma unroll
        for (int t = 0; t < T::TXT; ++t)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[t][j] = breg[j];
        constexpr int COLS = S * (T::TXT - 1) + 3;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
#pragma unroll
            for (int cx = 0; cx < COLS; ++cx) {
                const uint32_t a = src + (uint32_t) (((tyl * S + ky) * T::IW + txl * S + cx) * 128);
                uint32_t h[4], l[4];
                asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(h[0]), "=r"(h[1]), "=r"(h[2]), "=r"(h[3]) : "r"(a));
                asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(l[0]), "=r"(l[1]), "=r"(l[2]), "=r"(l[3]) : "r"(a + T::PLANE_BYTES));
                float v[8];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 vh = um_h2f(h[j]), vl = um_h2f(l[j]);
                    v[2 * j]     = vh.x + vl.x;
                    v[2 * j + 1] = vh.y + vl.y;
                }
#pragma unroll
                for (int t = 0; t < T::TXT; ++t) {
                    const int kx = cx - t * S; // compile-time after unrolling
                    if (kx >= 0 && kx < 3) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) acc[t][j] = fmaf(wreg[ky * 3 + kx][j], v[j], acc[t][j]);
                    }
                }
            }
        }
        const int oy = ty * T::TH + tyl;
        if (oy < p.OH && c < p.Cp) {
#pragma unroll
            for (int t = 0; t < T::TXT; ++t) {
                const int ox = tx * T::TW + txl + t;
                if (ox < p.OW) {
                    float v[8];
                    if (fast_act) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) v[j] = fminf(fmaxf(acc[t][j], acc[t][j] * slope), hi_clip);
                    } else {
#pragma unroll
                        for (int j = 0; j < 8; ++j) v[j] = umma_act_call(acc[t][j], p.act, p.alpha);
                    }
#pragma unroll
                    for (int j = 0; j < 8; ++j) v[j] = (c + j < p.C) ? v[j] : 0.0f; // channel padding stays zero
                    uint4 oh, ol;
                    um_split2(v[0], v[1], oh.x, ol.x);
                    um_split2(v[2], v[3], oh.y, ol.y);
                    um_split2(v[4], v[5], oh.z, ol.z);
                    um_split2(v[6], v[7], oh.w, ol.w);
                    const size_t o = (((size_t) n * p.OH + oy) * p.OW + ox) * p.Cp + c;
                    *reinterpret_cast<uint4*>(p.out_hi + o) = oh;
                    *reinterpret_cast<uint4*>(p.out_lo + o) = ol;
                }
            }
        }
        __syncthreads(); // everyone is done reading this stage
        if (tid == 0) {
            const int next = tile + DW_STAGES * gridDim.x;
            if (next < total) {
                fence_async_smem(); // generic-proxy reads above, async-proxy (TMA) writes below
                issue(next, stage);
            }
        }
    }
    (void) warp;
}

bool depthwise_tma_supported(const ConvArgs& a) {
    if (!a.in->lo || !a.out->lo) return false; // half-precision storage mode: the CUDA-core kernel (one plane)
    // tiles are 8x16 (stride 1) / 4x8 (stride 2) output pixels: tiny feature maps (7x7) would leave most of a tile empty
    const int tw = a.stride == 1 ? 16 : 8, th = a.stride == 1 ? 8 : 4;
    const int tx = (a.out->w + tw - 1) / tw, ty = (a.out->h + th - 1) / th;
    if ((double) a.out->w * a.out->h < 0.5 * (double) tx * tw * ty * th) return false;
    return a.k == 3 && (a.stride == 1 || a.stride == 2) && a.residual == nullptr && a.in->c == a.out->c && a.w->w_f32 != nullptr &&
           a.pad_mode <= SNNB_PAD_CONSTANT; // zero padding = the TMA out-of-bounds fill
}

template <int S> static int launch_depthwise_tma_s(snnb_context* ctx, const ConvArgs& a, EncodeTiledFn encode) {
    ctx->last_kernel = "depthwise_tma_kernel";
    using T = DwTile<S>;
    const snnb_tensor* in = a.in;
    snnb_tensor* out      = a.out;
    DwTmaParams p;
    p.out_hi = out->hi, p.out_lo = out->lo;
    p.w = a.w->w_f32, p.bias = a.w->bias;
    p.N = out->n, p.OH = out->h, p.OW = out->w, p.C = out->c, p.Cp = out->cp;
    p.pad_x = a.pad_x, p.pad_y = a.pad_y;
    p.tiles_x = (out->w + T::TW - 1) / T::TW, p.tiles_y = (out->h + T::TH - 1) / T::TH, p.chunks = (out->cp + 63) / 64;
    p.act = a.act, p.alpha = a.alpha;
    CUtensorMap tmI[2];
    {
        const cuuint64_t dims[4]    = {(cuuint64_t) in->c, (cuuint64_t) in->w, (cuuint64_t) in->h, (cuuint64_t) in->n}; // channels >= C read as zero
        const cuuint64_t strides[3] = {(cuuint64_t) in->cp * 2, (cuuint64_t) in->w * in->cp * 2, (cuuint64_t) in->h * in->w * in->cp * 2};
        const cuuint32_t box[4]     = {64, (cuuint32_t) T::IW, (cuuint32_t) T::IH, 1};
        const cuuint32_t estr[4]    = {1, 1, 1, 1};
        __half* planes[2]    = {in->hi, in->lo};
        for (int i = 0; i < 2; ++i) {
            CUresult r = encode(&tmI[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, planes[i], dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
            SNNB_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled(depthwise input) failed: %d", (int) r);
        }
    }
    if (ensure_smem_attr(ctx, (const void*) depthwise_tma_kernel<S>, S == 1 ? ATTR_DW1 : ATTR_DW2, T::SMEM_BYTES)) return 1;
    const long long total = (long long) p.N * p.tiles_y * p.tiles_x * p.chunks;
    const int grid        = (int) std::min<long long>(total, 2 * ctx->sm_count); // two CTAs per SM (128 registers, <= 93 KB of shared memory each)
    return launch_done(ctx, launch_k_pdl(depthwise_tma_kernel<S>, dim3(grid), dim3(DW_THREADS), T::SMEM_BYTES, ctx->stream, tmI[0], tmI[1], p),
                       S == 1 ? "depthwise_tma_kernel<1>" : "depthwise_tma_kernel<2>");
}

int launch_depthwise_tma(snnb_context* ctx, const ConvArgs& a) {
    EncodeTiledFn encode = get_encode(ctx);
    SNNB_REQUIRE(encode, "launch_depthwise_tma: cuTensorMapEncodeTiled is unavailable in this driver");
    return a.stride == 1 ? launch_depthwise_tma_s<1>(ctx, a, encode) : launch_depthwise_tma_s<2>(ctx, a, encode);
}

// The stream-K schedule exactly as the kernel's roles derive it (decode_work / sk_first_work / sk_next_work run on the host here), one row
// {cta, tile, kb0, kb1, piece, pieces} per work item in each CTA's order: lets the CPU test suite check the integer arithmetic
// (coverage, piece numbering, balance) without a GPU. Returns the number of rows, or -1 when nothing would be cut.
int streamk_schedule(int tiles, int num_kb, int sms, int* rows, int capacity) {
    UmmaParams p {};
    int dp = 0, ctas = 0;
    long long units = 0;
    if (tiles <= 0 || num_kb <= 0 || sms <= 0 || tiles % sms == 0 || !streamk_split(tiles, num_kb, sms, dp, units, ctas)) return -1;
    p.sk = 1, p.sk_dp = dp, p.sk_ctas = ctas, p.sk_units = units, p.ksplit = 1, p.kb_per_split = num_kb;
    const int grid = dp > 0 ? sms : ctas, end = dp + 4 * ctas;
    int n = 0;
    for (int cta = 0; cta < grid; ++cta)
        for (int work = sk_first_work(p, cta, end); work < end; work = sk_next_work(p, work, cta, grid, num_kb, end)) {
            const WorkItem w = decode_work<true>(p, work, tiles, num_kb);
            if (n < capacity) {
                int* r = rows + 6 * (size_t) n;
                r[0] = cta, r[1] = w.tile, r[2] = w.kb0, r[3] = w.kb1, r[4] = w.piece, r[5] = w.pieces;
            }
            ++n;
        }
    return n;
}

} // namespace snnb
