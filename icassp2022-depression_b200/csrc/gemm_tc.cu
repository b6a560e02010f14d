// gemm_tc.cu — tensor-core path of the time-parallel input projection (K1) and of the wgrad / dgrad GEMMs:
//     C[M,N] = A[M,K] * W[N,K]^T + bias          fp32 in / fp32 out, 3xTF32 on Hopper wgmma
//
// The hidden x input gate contraction over ALL time steps at once is the one genuinely dense GEMM of the path
// (M = B*T up to 15360, N = G*H, K = I), so it goes to the tensor cores — but the reference arithmetic is fp32
// (torch rnn.py:1221-1224 / :842-847) and parity is judged at 1e-5, which plain TF32 (10-bit mantissa) cannot hold.
// Each operand is therefore split x = hi + lo with hi = rna_tf32(x), lo = x - hi (exact), and three MMAs accumulate
// hi*hi + lo*hi + hi*lo (the dropped lo*lo term is ~2^-22 relative).
// The tensor core adds into its fp32 accumulator with truncation rather than round-to-nearest, a bias that grows with
// the number of MMAs chained on one accumulator. So the chain is cut after every k-block (12 MMAs): the wgmma
// accumulator restarts from zero and is added into a second register accumulator with ordinary round-to-nearest fp32.
// Resulting error ~1e-6 relative to the largest output, same order as fp32 FFMA.
//
// Kernel anatomy (one 128x128 output tile per CTA and work item, 384 threads, persistent over the tiles):
//   warpgroup 0   : producer — K-major operands (contraction index contiguous) arrive by TMA, 2-D tiles of
//                   128 rows x 32 fp32 in the 128-byte swizzle wgmma reads; MN-major operands (contraction index = the
//                   source's row index: dG, X, h_prev in the wgrads) are read with coalesced loads and written
//                   transposed into the same swizzled K-major layout, since wgmma takes tf32 operands K-major only.
//                   A 3-stage shared-memory ring (A_hi, A_lo, W_hi, W_lo per stage), mbarrier full/empty.
//                   fp32 A mode (the forward input projection): A arrives unsplit, 16 KB of fp32 per stage (the A_lo
//                   slot stays unused), by a 3-D TMA that reads the layer input in place (batch-first / permuted views
//                   included); one thread issues it with the W tiles.
//   warpgroups 1-2: consumers — 64 rows of the tile each: wgmma.m64n128k8.tf32, 12 per stage, then the
//                   round-to-nearest flush and finally the epilogue (+ folded biases, loaded before the first store).
//                   Presplit A: both operands from shared-memory descriptors. fp32 A: each thread loads its A fragment
//                   (16 floats per k-block), splits it in registers with the rounding of split_tf32_kernel and issues
//                   the MMAs with A from registers; the next k-block's fragment is loaded while the current MMAs run.
//                   The MMAs see exactly the operands of the presplit path, so C is bit-identical, while A is read
//                   from HBM / L2 in fp32 (half the bytes), never written back split, and read from shared memory
//                   once instead of three times per k-step. setmaxnreg moves registers from the producer (40) to the
//                   consumers (232) for the two fragment buffers.
//
// Single-pass TF32 (TF32 = true, B200RNN_FLAG_TF32: the caller follows torch's fp32 matmul precision "tf32"): one MMA
// per k-step, hi * hi, with every operand rounded to TF32 (cvt.rna) exactly once. The W_lo / A_lo tiles are neither
// written nor loaded (a stage carries 32 KB instead of 48 KB) and a k-block is 4 MMAs; the round-to-nearest flush after
// every k-block, the streamed publication and the epilogue are those of the 3xTF32 kernel.
#include <cuda.h>  // CUtensorMap types only; the encoder is fetched through cudaGetDriverEntryPoint
#include <cuda_fp16.h>
#include <mutex>
#include <stdlib.h>
#include <string.h>

#include "gemm_f32.cuh"
#include "gemm_h16_layout.cuh"
#include "h16.cuh"
#include "profile.cuh"
#include "ptx.cuh"
#include "rec_h16_layout.cuh"

namespace b200rnn {

namespace {

constexpr int BM = TC_TILE_M, BN = TC_TILE_N, BK = 32, STAGES = 3;
constexpr int LNB_BLOCKS = NUM_SMS * 2;  // CTAs of the LayerNorm backward (per-CTA column partials, reduced in fixed order)
constexpr int TILE_BYTES = BM * BK * 4;        // 16 KB, both A and W tiles (BM == BN)
constexpr int STAGE_BYTES = 4 * TILE_BYTES;    // A_hi, A_lo, W_hi, W_lo
constexpr int TC_THREADS = 384;
constexpr int TC_SMEM = STAGES * STAGE_BYTES + 1024 /*alignment slack*/ + 128 /*barriers*/;

// ---- PTX wrappers specific to this kernel -----------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          ptx::smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(ptx::smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// box of a 3-D map: coordinates (k, inner row, outer row)
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* map, int c0, int c1, int c2,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
          ptx::smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(ptx::smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// raise the expected transaction bytes of the current phase without arriving
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(ptx::smem_u32(bar)), "r"(bytes)
               : "memory");
}

// mbarrier phase wait that gives up after ~2^24 polls (seconds): in the native 16-bit kernel a TMA transaction that never
// completes (a map that disagrees with the expected bytes) becomes a trap, not a hang
__device__ __forceinline__ void bounded_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t n = 0; !ptx::mbar_try_wait(bar, parity); ++n)
    if (n > (1u << 24)) __trap();
}

// shared-memory matrix descriptor (sm_90): K-major tile, 128-byte swizzle, rows of 128 B, 8-row groups 1024 B apart
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);  // start address        [0,14)
  d |= (uint64_t)1 << 16;                       // leading byte offset  (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;             // stride byte offset: 8 rows * 128 B
  d |= (uint64_t)1 << 62;                       // layout type: SWIZZLE_128B
  return d;
}

#define B200_ACC8(i) "+f"(d[i + 0]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), \
                     "+f"(d[i + 6]), "+f"(d[i + 7])
// D[64x128] (+)= A[64x8] * B[128x8]^T, tf32 operands from shared memory, fp32 accumulator in registers
__device__ __forceinline__ void wgmma_tf32_m64n128k8(float (&d)[64], uint64_t adesc, uint64_t bdesc, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}"
      : B200_ACC8(0), B200_ACC8(8), B200_ACC8(16), B200_ACC8(24), B200_ACC8(32), B200_ACC8(40), B200_ACC8(48),
        B200_ACC8(56)
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// the same with A from registers: a[0..3] = A(g, t), A(g + 8, t), A(g, t + 4), A(g + 8, t + 4) of the warp's 16 rows,
// g = lane / 4, t = lane % 4 (tf32 bit patterns)
__device__ __forceinline__ void wgmma_tf32_m64n128k8_ra(float (&d)[64], const uint32_t* a, uint64_t bdesc,
                                                        int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : B200_ACC8(0), B200_ACC8(8), B200_ACC8(16), B200_ACC8(24), B200_ACC8(32), B200_ACC8(40), B200_ACC8(48),
        B200_ACC8(56)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
// D[64x128] (+)= A[64x16] * B[128x16]^T in fp16 with fp32 accumulation, A from registers: a[r] = f16x2 of
// A(g + 8 (r & 1), 2t + 8 (r >> 1) + {0, 1}) of the warp's 16 rows (low half first), B K-major from shared memory
__device__ __forceinline__ void wgmma_f16_m64n128k16_ra(float (&d)[64], const uint32_t* a, uint64_t bdesc,
                                                        int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : B200_ACC8(0), B200_ACC8(8), B200_ACC8(16), B200_ACC8(24), B200_ACC8(32), B200_ACC8(40), B200_ACC8(48),
        B200_ACC8(56)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
// the same in f16 (BF = false) or bf16 (BF = true) with both the A fragment (layout of wgmma_f16_m64n128k16_ra) and
// B from 16-bit data as it lies: the native 16-bit input projection (gemm_n16_kernel)
template <bool BF>
__device__ __forceinline__ void wgmma_n16_m64n128k16_ra(float (&d)[64], const uint32_t* a, uint64_t bdesc,
                                                        int accumulate) {
  if constexpr (BF)
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %69, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
        : B200_ACC8(0), B200_ACC8(8), B200_ACC8(16), B200_ACC8(24), B200_ACC8(32), B200_ACC8(40), B200_ACC8(48),
          B200_ACC8(56)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
  else
    wgmma_f16_m64n128k16_ra(d, a, bdesc, accumulate);
}
#undef B200_ACC8
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of the accumulator across the asynchronous MMA
__device__ __forceinline__ void reg_fence(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

struct TcArgs {
  float* C;
  RowMap c_rows;
  int M, N, K;
  const float* bias1;
  const float* bias2;
  int bias2_n;
  int tiles_m, tiles_n;
  int accumulate;   // C += result (splitk == 1 only)
  int a_mn, b_mn;   // operand is MN-major: source matrix [K rows][M or N contiguous] (wgrad / dgrad without transposes)
  const float *a_hi, *a_lo, *b_hi, *b_lo;  // MN-major operands are read through these (K-major ones through TMA)
  long long lda, ldb;
  int splitk;       // > 1: work item = (k-split, tile); raw partial sums go to partial[ks][M][N]
  int kb_per_split; // k-blocks per split
  float* partial;
  int* ready;       // streamed (splitk == 1): tiles walked time-major, ready[m] += 1 per finished tile of row tile m
  int a_f32;        // A is fp32 (map_a_hi, 3-D), split in registers by the consumers; W K-major presplit
  int a_inner;      // fp32 A: rows per outer index of the 3-D map (tile m0 sits at (m0 % a_inner, m0 / a_inner))
  int tf32;         // single-pass TF32: the lo operands are absent (host side only: selects the kernel instantiation)
  const int* w_exp; // fp16 pairs: e_n of every W row (gemm_h16_layout.cuh), the epilogue scales column n by 2^-e_n
  int f16;          // fp16 pairs (gemm_f16x3_kernel; host side only)
  int n16;          // native 16-bit operands: TC_F16 or TC_BF16 (gemm_n16_kernel; host side only), else 0
};

// the arithmetic of one instantiation: 3xTF32, single-pass TF32, fp16 (hi, lo) pairs (fp32 A only), or native f16 /
// bf16 operands (16-bit A and W, one MMA per k-step)
enum TcMath { TC_3XTF32, TC_TF32, TC_F16X3, TC_F16, TC_BF16 };

constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;  // 128 x 40 + 256 x 232 <= 64K registers of the SM

// work item -> output tile origin: m fastest (consecutive tiles of a CTA mostly share their W tile rows in L2), or
// time-major when streamed (the consumer reads row tile m after m - 1)
__device__ __forceinline__ void tile_origin(const TcArgs& a, int tile, int& m0, int& n0) {
  if (a.ready) {
    m0 = (tile / a.tiles_n) * BM;
    n0 = (tile % a.tiles_n) * BN;
  } else {
    m0 = (tile % a.tiles_m) * BM;
    n0 = (tile / a.tiles_m) * BN;
  }
}

// One 128 x BK tile of an MN-major operand (src: [K rows][ext columns], leading dimension ld) into the K-major
// 128-byte-swizzled layout: thread t owns tile row t (= source column c0 + t), its 32 k values go out as 8 float4
// chunks, chunk j at ((j ^ (t & 7)) * 16) inside the 128-byte row. Rows / columns past the source read as zero.
__device__ __forceinline__ void load_mn_tile(unsigned char* tile, const float* __restrict__ src, long long ld, int ext,
                                             int K, int c0, int k0, int t) {
  const int c = c0 + t;
  float v[BK];
#pragma unroll
  for (int kk = 0; kk < BK; ++kk)
    v[kk] = (c < ext && k0 + kk < K) ? __ldg(src + (long long)(k0 + kk) * ld + c) : 0.f;
  unsigned char* row = tile + (t >> 3) * 1024 + (t & 7) * 128;
#pragma unroll
  for (int j = 0; j < BK / 4; ++j)
    *reinterpret_cast<float4*>(row + ((j ^ (t & 7)) << 4)) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
}

// Persistent: each CTA walks work items blockIdx.x, +gridDim.x, ... (tile_origin). Producer and consumers loop
// independently over the same item sequence and meet only through the full / empty mbarriers of the shared-memory ring.
// Streamed (args.ready, api.cu): the kernel lets the next kernel of the stream launch at once (griddepcontrol), and
// after a tile's stores the consumer warpgroups publish it with one release increment of ready[m]. Every read of the
// A operand of a tile precedes that increment (the consumers have drained the ring stages of the tile), and the kernel
// itself never waits on anything outside its CTA.
// MN: some operand is MN-major (backward wgrad / dgrad). Its producer keeps 32 loads per thread in flight and needs
// the default register budget, so that instantiation has no setmaxnreg; in the K-major one (every operand by TMA, one
// thread issues) the producer gives registers to the consumers, whose fp32-A path holds the running sum, the wgmma
// accumulator and two A fragments (4 x 64 registers).
// fp16 pairs (MATH = TC_F16X3, gemm_f16x3_kernel; fp32 A only): a k-block is 64 k (KB), A arrives as two boxes of 32
// (ring slots 0 and 1), W as fp16 hi / lo tiles of 128 rows x 128 bytes (slots 2 and 3) with their row exponents in
// args.w_exp (gemm_h16_layout.cuh). Each consumer scales its rows of the k-block's A by 2^e_m (h16::scale_exp of the
// row's max |a| over the k-block), splits them into fp16 hi / lo in registers and runs lo*hi, hi*lo, hi*hi as
// wgmma.m64n128k16 (12 per k-block); the drain unscales with total = fma(acc, 2^-e_m, total), the epilogue multiplies
// column n by 2^-e_n before the biases.
// Native 16-bit (MATH = TC_F16 / TC_BF16, gemm_n16_kernel; args.a_f32 = 1 for the single TMA issuer): a k-block is 64 k,
// A (128 rows x 128 bytes, 3-D map read in place) in slot 0 and W in slot 2, both K-major under the 128-byte swizzle;
// each consumer loads its A fragment of the k-block as it lies (the fp32-A kernel's addressing, 16 registers) and runs
// 4 wgmma.m64n128k16 with W from shared memory, then the round-to-nearest drain of the 3xTF32 kernel. No split, no
// scale: the products are exact in fp32.
template <bool MN, int MATH>
__device__ __forceinline__ void gemm_tc_body(const CUtensorMap& map_a_hi, const CUtensorMap& map_a_lo,
                                             const CUtensorMap& map_b_hi, const CUtensorMap& map_b_lo,
                                             const TcArgs args) {
  constexpr bool TF32 = MATH == TC_TF32, F16 = MATH == TC_F16X3;
  constexpr bool NAT = MATH == TC_F16 || MATH == TC_BF16;
  constexpr int KB = (F16 || NAT) ? g16::BK : BK;  // k per ring stage
  extern __shared__ unsigned char smem_raw[];
  // aligned by offset so that the compiler keeps the shared state space (LDS/STS instead of generic LD/ST)
  unsigned char* base = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(base + STAGES * STAGE_BYTES);
  uint64_t* empty = full + STAGES;

  // canonical warp index: the shuffle makes it warp-uniform for the compiler, so the single-thread TMA issue stays on
  // the uniform datapath (no per-instruction R2UR broadcast loop around UTMALDG)
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int nkb_total = (args.K + KB - 1) / KB;  // the K tail reads as zero
  const int ntiles = args.tiles_m * args.tiles_n;
  const int nitems = ntiles * args.splitk;
  if (args.ready) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full[s], args.a_f32 ? 1 : 128);  // the TMA issuer (fp32 A) / every producer thread
      ptx::mbar_init(&empty[s], 8);                     // one arrival per consumer warp
    }
    ptx::fence_mbar_init();
    if (!args.a_mn) {
      prefetch_tmap(&map_a_hi);
      if (!TF32 && !args.a_f32) prefetch_tmap(&map_a_lo);
    }
    if (!args.b_mn) {
      prefetch_tmap(&map_b_hi);
      if (!TF32 && !NAT) prefetch_tmap(&map_b_lo);
    }
  }
  __syncthreads();

  if (warp < 4) {
    if constexpr (!MN) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
    const int t = threadIdx.x;
    if (F16 || (!MN && args.a_f32)) {  // one thread issues the fp32 A tile and the W tiles; the consumers split A
      if (warp == 0) {
        int it = 0;  // running k-block counter across items (ring position)
        for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
          int m0, n0;
          tile_origin(args, item % ntiles, m0, n0);
          for (int kb = 0; kb < nkb_total; ++kb, ++it) {
            const int s = it % STAGES;
            if constexpr (NAT)
              bounded_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
            else
              ptx::mbar_wait(&empty[s], ((it / STAGES) & 1) ^ 1);
            unsigned char* st = base + s * STAGE_BYTES;
            if (ptx::elect_one_sync()) {  // 3xTF32 / TF32: the A_lo slot stays unused (A is split in registers);
                                          // fp16 pairs: it holds the second 32 k of A
              ptx::mbar_arrive_expect_tx(&full[s], (NAT ? 2u : F16 ? 4u : TF32 ? 2u : 3u) * TILE_BYTES);
              tma_load_3d(st + 0 * TILE_BYTES, &map_a_hi, kb * KB, m0 % args.a_inner, m0 / args.a_inner, &full[s]);
              if (F16)
                tma_load_3d(st + 1 * TILE_BYTES, &map_a_hi, kb * KB + BK, m0 % args.a_inner, m0 / args.a_inner,
                            &full[s]);
              tma_load_2d(st + 2 * TILE_BYTES, &map_b_hi, kb * KB, n0, &full[s]);
              if (!TF32 && !NAT) tma_load_2d(st + 3 * TILE_BYTES, &map_b_lo, kb * KB, n0, &full[s]);
            }
            __syncwarp();
          }
        }
      }
    } else {
      const bool a_mn = MN && args.a_mn, b_mn = MN && args.b_mn;
      constexpr uint32_t parts = TF32 ? 1u : 2u;  // hi (and lo) tile per operand
      const uint32_t tx = (a_mn ? 0u : parts * TILE_BYTES) + (b_mn ? 0u : parts * TILE_BYTES);
      int it = 0;  // running k-block counter across items (ring position)
      for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
        const int tile = item % ntiles, ks = item / ntiles;
        int m0, n0;
        tile_origin(args, tile, m0, n0);
        const int kb0 = ks * args.kb_per_split;
        const int kb1 = min(nkb_total, kb0 + args.kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const int s = it % STAGES;
          const uint32_t ph = (it / STAGES) & 1;
          ptx::mbar_wait(&empty[s], ph ^ 1);
          unsigned char* st = base + s * STAGE_BYTES;
          if (warp == 0 && tx) {
            if (ptx::elect_one_sync()) {
              mbar_expect_tx(&full[s], tx);
              if (!a_mn) {
                tma_load_2d(st + 0 * TILE_BYTES, &map_a_hi, kb * BK, m0, &full[s]);
                if (!TF32) tma_load_2d(st + 1 * TILE_BYTES, &map_a_lo, kb * BK, m0, &full[s]);
              }
              if (!b_mn) {
                tma_load_2d(st + 2 * TILE_BYTES, &map_b_hi, kb * BK, n0, &full[s]);
                if (!TF32) tma_load_2d(st + 3 * TILE_BYTES, &map_b_lo, kb * BK, n0, &full[s]);
              }
            }
            __syncwarp();
          }
          if (a_mn) {
            load_mn_tile(st + 0 * TILE_BYTES, args.a_hi, args.lda, args.M, args.K, m0, kb * BK, t);
            if (!TF32) load_mn_tile(st + 1 * TILE_BYTES, args.a_lo, args.lda, args.M, args.K, m0, kb * BK, t);
          }
          if (b_mn) {
            load_mn_tile(st + 2 * TILE_BYTES, args.b_hi, args.ldb, args.N, args.K, n0, kb * BK, t);
            if (!TF32) load_mn_tile(st + 3 * TILE_BYTES, args.b_lo, args.ldb, args.N, args.K, n0, kb * BK, t);
          }
          if (a_mn || b_mn) ptx::fence_proxy_async();  // generic stores -> visible to wgmma (async proxy)
          ptx::mbar_arrive(&full[s]);
        }
      }
    }
  } else {
    if constexpr (!MN) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
    const int wg = (threadIdx.x >> 7) - 1;   // consumer warpgroup: tile rows [64 wg, 64 wg + 64)
    const int wq = warp & 3;                 // warp within the warpgroup: 16 accumulator rows each
    // the 12 (TF32: 4) MMAs of the k-block in ring position `pos` into acc, which restarts from zero; committed as one
    // group
    auto issue = [&](float (&acc)[64], int pos) {
      ptx::mbar_wait(&full[pos % STAGES], (pos / STAGES) & 1);
      const uint32_t st = ptx::smem_u32(base + (pos % STAGES) * STAGE_BYTES);
      const uint64_t a_hi = make_kmajor_sw128_desc(st + 0 * TILE_BYTES + wg * 8192);
      const uint64_t a_lo = make_kmajor_sw128_desc(st + 1 * TILE_BYTES + wg * 8192);
      const uint64_t b_hi = make_kmajor_sw128_desc(st + 2 * TILE_BYTES);
      const uint64_t b_lo = make_kmajor_sw128_desc(st + 3 * TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 8; ++k) {
        const uint64_t adv = (uint64_t)(k * (32 >> 4));  // K step of 8 tf32 = 32 bytes inside the swizzle atom
        if constexpr (TF32) {
          wgmma_tf32_m64n128k8(acc, a_hi + adv, b_hi + adv, k != 0);
        } else {
          wgmma_tf32_m64n128k8(acc, a_lo + adv, b_hi + adv, k != 0);
          wgmma_tf32_m64n128k8(acc, a_hi + adv, b_lo + adv, 1);
          wgmma_tf32_m64n128k8(acc, a_hi + adv, b_hi + adv, 1);
        }
      }
      wgmma_commit();
    };
    // k-block `pos` has completed: hand its stage back and add it into total (round-to-nearest, increasing kb)
    auto drain = [&](float (&total)[64], float (&acc)[64], int pos) {
      reg_fence(acc);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&empty[pos % STAGES]);  // this warp's share of the stage has been read
#pragma unroll
      for (int i = 0; i < 64; ++i) total[i] += acc[i];
    };
    // fp32 A: this thread's A fragment of the k-block in ring position `pos` (rows g and g + 8 of the warp's 16, k = t + 4j
    // of the 32; conflict-free under the 128-byte swizzle since row & 7 == g), split as split_tf32_kernel does:
    // fa[8 s + i] = hi of a_i at k-step s, fa[8 s + 4 + i] = lo; TF32: fa[4 s + i] = hi, the rest unused
    const int g = lane >> 2, tq = lane & 3;
    const uint32_t a_row = (uint32_t)(wg * 64 + wq * 16 + g) * 128u + tq * 4u;
    auto load_a = [&](uint32_t (&fa)[32], int pos) {
      ptx::mbar_wait(&full[pos % STAGES], (pos / STAGES) & 1);
      const unsigned char* at = base + (pos % STAGES) * STAGE_BYTES + a_row;
#pragma unroll
      for (int s4 = 0; s4 < BK / 8; ++s4) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float x = *reinterpret_cast<const float*>(at + (i & 1) * 1024 + ((((2 * s4 + (i >> 1)) ^ g)) << 4));
          uint32_t h;
          asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
          if constexpr (TF32) {
            fa[4 * s4 + i] = h;
          } else {
            fa[8 * s4 + i] = h;
            fa[8 * s4 + 4 + i] = __float_as_uint(x - __uint_as_float(h));
          }
        }
      }
    };
    // the 12 (TF32: 4) MMAs of a k-block with A from registers: same products, same order as `issue`
    auto issue_ra = [&](float (&acc)[64], const uint32_t (&fa)[32], int pos) {
      const uint32_t st = ptx::smem_u32(base + (pos % STAGES) * STAGE_BYTES);
      const uint64_t b_hi = make_kmajor_sw128_desc(st + 2 * TILE_BYTES);
      const uint64_t b_lo = make_kmajor_sw128_desc(st + 3 * TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 8; ++k) {
        const uint64_t adv = (uint64_t)(k * (32 >> 4));
        if constexpr (TF32) {
          wgmma_tf32_m64n128k8_ra(acc, &fa[4 * k], b_hi + adv, k != 0);
        } else {
          wgmma_tf32_m64n128k8_ra(acc, &fa[8 * k + 4], b_hi + adv, k != 0);
          wgmma_tf32_m64n128k8_ra(acc, &fa[8 * k], b_lo + adv, 1);
          wgmma_tf32_m64n128k8_ra(acc, &fa[8 * k], b_hi + adv, 1);
        }
      }
      wgmma_commit();
    };
    // fp16 pairs: this thread's A fragment of the 64 k of ring position `pos`, rows g and g + 8, k = 16 s + 8 j + 2 tq
    // + {0, 1} (float2 loads, conflict-free under the swizzle). Each row is scaled by 2^e, e = h16::scale_exp of its
    // max |a| over the k-block (quad max: the 4 lanes of a row hold its 64 k), and split; fa[8 s + r] = hi, fa[8 s + 4 +
    // r] = lo of register r = h + 2 j of k-step s; sc[h] = 2^-e of row g + 8 h
    const uint32_t a_row16 = (uint32_t)(wg * 64 + wq * 16 + g) * 128u + (tq & 1) * 8u;
    auto load_a16 = [&](uint32_t (&fa)[32], float (&sc)[2], int pos) {
      ptx::mbar_wait(&full[pos % STAGES], (pos / STAGES) & 1);
      const unsigned char* at = base + (pos % STAGES) * STAGE_BYTES + a_row16;
      float x[2][16];  // [h][4 s + 2 j + e]
#pragma unroll
      for (int s4 = 0; s4 < 4; ++s4)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const float2 v = *reinterpret_cast<const float2*>(
                at + (s4 >> 1) * TILE_BYTES + h * 1024 + (((4 * (s4 & 1) + 2 * j + (tq >> 1)) ^ g) << 4));
            x[h][4 * s4 + 2 * j] = v.x;
            x[h][4 * s4 + 2 * j + 1] = v.y;
          }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float m = 0.f;
#pragma unroll
        for (int i = 0; i < 16; ++i) m = fmaxf(m, fabsf(x[h][i]));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
        const int e = g16::scale_exp_bits(m);
        const float up = g16::exp2i(e);
        sc[h] = g16::exp2i(-e);
#pragma unroll
        for (int i = 0; i < 16; ++i) x[h][i] *= up;
      }
#pragma unroll
      for (int s4 = 0; s4 < 4; ++s4)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float x0 = x[h][4 * s4 + 2 * j], x1 = x[h][4 * s4 + 2 * j + 1];
            const __half2 hi = __floats2half2_rn(x0, x1);
            const __half2 lo = __floats2half2_rn(x0 - __low2float(hi), x1 - __high2float(hi));
            fa[8 * s4 + h + 2 * j] = *reinterpret_cast<const uint32_t*>(&hi);
            fa[8 * s4 + 4 + h + 2 * j] = *reinterpret_cast<const uint32_t*>(&lo);
          }
    };
    // the 12 fp16 MMAs of a k-block: per k-step of 16 lo*hi, hi*lo, hi*hi, as the 3xTF32 k-block orders them
    auto issue_ra16 = [&](float (&acc)[64], const uint32_t (&fa)[32], int pos) {
      const uint32_t st = ptx::smem_u32(base + (pos % STAGES) * STAGE_BYTES);
      const uint64_t b_hi = make_kmajor_sw128_desc(st + 2 * TILE_BYTES);
      const uint64_t b_lo = make_kmajor_sw128_desc(st + 3 * TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < g16::BK / 16; ++k) {
        const uint64_t adv = (uint64_t)(k * (32 >> 4));  // K step of 16 f16 = 32 bytes inside the swizzle atom
        wgmma_f16_m64n128k16_ra(acc, &fa[8 * k + 4], b_hi + adv, k != 0);
        wgmma_f16_m64n128k16_ra(acc, &fa[8 * k], b_lo + adv, 1);
        wgmma_f16_m64n128k16_ra(acc, &fa[8 * k], b_hi + adv, 1);
      }
      wgmma_commit();
    };
    // native 16-bit: the 4 MMAs of a k-block of 64. Register 4 s + i of the A fragment holds the pair at row g + 8 (i & 1),
    // k = 16 s + 8 (i >> 1) + 2 tq: 16-byte chunk 2 s + (i >> 1) of the row, swizzled by g, 4 tq bytes in (a_row)
    auto issue_n16 = [&](float (&acc)[64], int pos) {
      bounded_wait(&full[pos % STAGES], (pos / STAGES) & 1);
      const unsigned char* at = base + (pos % STAGES) * STAGE_BYTES + a_row;
      uint32_t fa[16];
#pragma unroll
      for (int s4 = 0; s4 < 4; ++s4)
#pragma unroll
        for (int i = 0; i < 4; ++i)
          fa[4 * s4 + i] = *reinterpret_cast<const uint32_t*>(at + (i & 1) * 1024 + (((2 * s4 + (i >> 1)) ^ g) << 4));
      const uint64_t b = make_kmajor_sw128_desc(ptx::smem_u32(base + (pos % STAGES) * STAGE_BYTES) + 2 * TILE_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < g16::BK / 16; ++k) {
        const uint64_t adv = (uint64_t)(k * (32 >> 4));  // K step of 16 halves = 32 bytes inside the swizzle atom
        wgmma_n16_m64n128k16_ra<MATH == TC_BF16>(acc, &fa[4 * k], b + adv, k != 0);
      }
      wgmma_commit();
    };
    // fp16 pairs: as drain, the k-block's sum unscaled by its rows' 2^-e_m in the same rounding
    auto drain16 = [&](float (&total)[64], float (&acc)[64], const float (&sc)[2], int pos) {
      reg_fence(acc);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&empty[pos % STAGES]);
#pragma unroll
      for (int i = 0; i < 64; ++i) total[i] = fmaf(acc[i], sc[(i >> 1) & 1], total[i]);
    };
    int it = 0;
    for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
      const int tile = item % ntiles, ks = item / ntiles;
      const int nkb = min(nkb_total, (ks + 1) * args.kb_per_split) - ks * args.kb_per_split;
      int m0, n0;
      tile_origin(args, tile, m0, n0);
      float total[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) total[i] = 0.f;
      float acc[64];
      if constexpr (NAT) {
        for (int kb = 0; kb < nkb; ++kb) {
          issue_n16(acc, it + kb);
          wgmma_wait0();
          drain(total, acc, it + kb);
        }
      } else if (F16 || (!MN && args.a_f32)) {
        // A from registers: the k-block's fp32 fragment is loaded and split here; the next k-block's is loaded while
        // the current MMAs run. Fragments alternate between fa0 and fa1; the loop body is unconditional and the tail
        // peeled, so no branch merges registers a wgmma in flight reads.
        uint32_t fa0[32], fa1[32];
        if constexpr (F16) {  // the same schedule; each fragment carries its rows' unscales
          float sc0[2], sc1[2];
          load_a16(fa0, sc0, it);
          int kb = 0;
          for (; kb + 2 < nkb; kb += 2) {
            issue_ra16(acc, fa0, it + kb);
            load_a16(fa1, sc1, it + kb + 1);
            wgmma_wait0();
            drain16(total, acc, sc0, it + kb);
            issue_ra16(acc, fa1, it + kb + 1);
            load_a16(fa0, sc0, it + kb + 2);
            wgmma_wait0();
            drain16(total, acc, sc1, it + kb + 1);
          }
          issue_ra16(acc, fa0, it + kb);
          if (kb + 1 < nkb) load_a16(fa1, sc1, it + kb + 1);
          wgmma_wait0();
          drain16(total, acc, sc0, it + kb);
          if (kb + 1 < nkb) {
            issue_ra16(acc, fa1, it + kb + 1);
            wgmma_wait0();
            drain16(total, acc, sc1, it + kb + 1);
          }
        } else {
          load_a(fa0, it);
          int kb = 0;
          for (; kb + 2 < nkb; kb += 2) {
            issue_ra(acc, fa0, it + kb);
            load_a(fa1, it + kb + 1);
            wgmma_wait0();
            drain(total, acc, it + kb);
            issue_ra(acc, fa1, it + kb + 1);
            load_a(fa0, it + kb + 2);
            wgmma_wait0();
            drain(total, acc, it + kb + 1);
          }
          issue_ra(acc, fa0, it + kb);
          if (kb + 1 < nkb) load_a(fa1, it + kb + 1);
          wgmma_wait0();
          drain(total, acc, it + kb);
          if (kb + 1 < nkb) {
            issue_ra(acc, fa1, it + kb + 1);
            wgmma_wait0();
            drain(total, acc, it + kb + 1);
          }
        }
      } else {
        for (int kb = 0; kb < nkb; ++kb) {
          issue(acc, it + kb);
          wgmma_wait0();
          drain(total, acc, it + kb);
        }
      }
      it += nkb;
      // accumulator fragment: element i sits at row 16 wq + lane/4 + 8 ((i/2) & 1), column 8 (i/4) + 2 (lane%4) + i%2
      const int r0 = m0 + wg * 64 + wq * 16 + (lane >> 2);
      // the biases of this thread's 32 columns, loaded before the first store: loads placed after a store of C would
      // each wait a full load latency (the compiler cannot move them across a store that might alias)
      float b1v[32], b2v[32], wsc[32];  // wsc: fp16 pairs, 2^-e_n of the columns
#pragma unroll
      for (int q = 0; q < 16; ++q) {
        const int n = n0 + 8 * q + 2 * (lane & 3);
        if constexpr (F16) {
          wsc[2 * q] = g16::exp2i(-__ldg(args.w_exp + n));
          wsc[2 * q + 1] = g16::exp2i(-__ldg(args.w_exp + n + 1));
        }
        b1v[2 * q] = b1v[2 * q + 1] = b2v[2 * q] = b2v[2 * q + 1] = 0.f;
        if (args.splitk == 1 && args.bias1) { b1v[2 * q] = __ldg(args.bias1 + n); b1v[2 * q + 1] = __ldg(args.bias1 + n + 1); }
        if (args.splitk == 1 && args.bias2) {
          if (n < args.bias2_n) b2v[2 * q] = __ldg(args.bias2 + n);
          if (n + 1 < args.bias2_n) b2v[2 * q + 1] = __ldg(args.bias2 + n + 1);
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        if (row >= args.M) continue;
        float* crow = (args.splitk > 1) ? args.partial + ((size_t)ks * args.M + row) * args.N + n0
                                        : args.C + args.c_rows.off(row) + n0;
#pragma unroll
        for (int q = 0; q < 16; ++q) {
          const int col = 8 * q + 2 * (lane & 3);
          float2 o = make_float2(total[4 * q + 2 * h], total[4 * q + 2 * h + 1]);
          if constexpr (F16) {
            o.x *= wsc[2 * q];
            o.y *= wsc[2 * q + 1];
          }
          if (args.splitk == 1) {
            const int n = n0 + col;
            if (args.bias1) { o.x += b1v[2 * q]; o.y += b1v[2 * q + 1]; }
            if (args.bias2) {
              if (n < args.bias2_n) o.x += b2v[2 * q];
              if (n + 1 < args.bias2_n) o.y += b2v[2 * q + 1];
            }
            if (args.accumulate) {
              const float2 old = *reinterpret_cast<const float2*>(crow + col);
              o.x += old.x; o.y += old.y;
            }
          }
          *reinterpret_cast<float2*>(crow + col) = o;
        }
      }
      if (args.ready) {  // publish the tile: every storing thread fences, the 256 consumer threads meet, one releases
        __threadfence();
        ptx::named_barrier_sync(1, 256);
        if (threadIdx.x == 128)
          asm volatile("red.release.gpu.global.add.s32 [%0], 1;" ::"l"(args.ready + m0 / BM) : "memory");
      }
    }
  }
}

template <bool MN, bool TF32>
__global__ void __launch_bounds__(TC_THREADS, 1)
    gemm_tf32x3_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                       const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
                       const TcArgs args) {
  gemm_tc_body<MN, TF32 ? TC_TF32 : TC_3XTF32>(map_a_hi, map_a_lo, map_b_hi, map_b_lo, args);
}

// fp32 A read in place and split into fp16 pairs on chip, W presplit into fp16 pairs (split_w16_kernel)
__global__ void __launch_bounds__(TC_THREADS, 1)
    gemm_f16x3_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_unused,
                      const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                      const TcArgs args) {
  gemm_tc_body<false, TC_F16X3>(map_a, map_unused, map_w_hi, map_w_lo, args);
}

// 16-bit A read in place and 16-bit W, both straight into wgmma (MATH = TC_F16 or TC_BF16)
template <int MATH>
__global__ void __launch_bounds__(TC_THREADS, 1)
    gemm_n16_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_unused,
                    const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_unused2,
                    const TcArgs args) {
  gemm_tc_body<false, MATH>(map_a, map_unused, map_w, map_unused2, args);
}

// W [N][K] (rows through `rows`) -> fp16 pairs (gemm_h16_layout.cuh): row n scaled by 2^e_n, e_n = h16::scale_exp of
// its max |w| (rec_h16_layout.cuh: a zero or non-finite row keeps e = 0), hi = RN_f16, lo = RN_f16(w 2^e_n - hi).
// One warp per row; K even.
__global__ void split_w16_kernel(const float* __restrict__ src, RowMap rows, int N, int K, __half* __restrict__ hi,
                                 __half* __restrict__ lo, int* __restrict__ exps) {
  const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
  for (int n = blockIdx.x * wpb + (threadIdx.x >> 5); n < N; n += gridDim.x * wpb) {
    const float* p = src + rows.off(n);
    float m = 0.f;
    for (int k = lane; k < K; k += 32) m = fmaxf(m, fabsf(__ldg(p + k)));
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    const int e = h16::scale_exp(m);
    const float up = ldexpf(1.f, e);
    for (int k = 2 * lane; k < K; k += 64) {
      const float x0 = __ldg(p + k) * up, x1 = __ldg(p + k + 1) * up;
      const __half2 h = __floats2half2_rn(x0, x1);
      *reinterpret_cast<__half2*>(hi + (size_t)n * K + k) = h;
      *reinterpret_cast<__half2*>(lo + (size_t)n * K + k) = __floats2half2_rn(x0 - __low2float(h), x1 - __high2float(h));
    }
    if (lane == 0) exps[n] = e;
  }
}

// x = hi + lo with hi = round-to-nearest TF32 (kept in a 32-bit container), lo = x - hi (exact in fp32).
// Reads rows through a RowMap (batch_first / permuted inputs), writes two dense [M,K] matrices (lo == NULL: hi only,
// the operand of a single-pass TF32 GEMM).
__global__ void split_tf32_kernel(const float* __restrict__ src, RowMap rows, int M, int K, float* __restrict__ hi,
                                  float* __restrict__ lo, int vec_ok) {
  const size_t nvec = (size_t)M * (K / 4);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    const int m = (int)(i / (K / 4));
    const int k = (int)(i - (size_t)m * (K / 4)) * 4;
    const float* p = src + rows.off(m) + k;
    float4 x;
    if (vec_ok) {
      x = __ldg(reinterpret_cast<const float4*>(p));
    } else {
      x = make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3));
    }
    float4 h, l;
    uint32_t t;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(x.x)); h.x = __uint_as_float(t); l.x = x.x - h.x;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(x.y)); h.y = __uint_as_float(t); l.y = x.y - h.y;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(x.z)); h.z = __uint_as_float(t); l.z = x.z - h.z;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(x.w)); h.w = __uint_as_float(t); l.w = x.w - h.w;
    *reinterpret_cast<float4*>(hi + (size_t)m * K + k) = h;
    if (lo) *reinterpret_cast<float4*>(lo + (size_t)m * K + k) = l;
  }
}

// Dense fp32 copy of a layer input whose rows the fp32-A GEMM cannot read in place (a batch size that neither divides
// 128 nor is a multiple of it, or misaligned strides); also zeroes `clear` (ready counters of a streamed GEMM).
__global__ void gather_rows_kernel(const float* __restrict__ src, RowMap rows, int M, int K, float* __restrict__ dst,
                                   int vec_ok, int* __restrict__ clear, int nclear) {
  if (blockIdx.x == 0)
    for (int i = threadIdx.x; i < nclear; i += blockDim.x) clear[i] = 0;
  const size_t nvec = (size_t)M * (K / 4);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    const int m = (int)(i / (K / 4));
    const int k = (int)(i - (size_t)m * (K / 4)) * 4;
    const float* p = src + rows.off(m) + k;
    const float4 x = vec_ok ? __ldg(reinterpret_cast<const float4*>(p)) : make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3));
    *reinterpret_cast<float4*>(dst + (size_t)m * K + k) = x;
  }
}

// LayerNorm(row) * gamma + beta — the prologue of audio_gru_whole.py:104 / fuse_net_whole.py:360, written dense in fp32
// as the A operand of K1 (which splits it on chip) and, when saved, of the layer-0 wgrad. One warp per row;
// Cc % 128 == 0, Cc <= 1024.
template <int NV>  // float4 per lane
__global__ void layernorm_kernel(const float* __restrict__ src, RowMap rows, int R, int Cc,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                 float* __restrict__ out, int* __restrict__ clear, int nclear,
                                 const int* __restrict__ lengths, int B) {
  if (blockIdx.x == 0)
    for (int i = threadIdx.x; i < nclear; i += blockDim.x) clear[i] = 0;
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < R; r += gridDim.x * wpb) {
    if (lengths && r / B >= __ldg(lengths + r % B)) {  // padding of a ragged batch: 0, whatever x holds there
#pragma unroll
      for (int i = 0; i < NV; ++i)
        *reinterpret_cast<float4*>(out + (size_t)r * Cc + i * 128 + lane * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
      continue;
    }
    const float* p = src + rows.off(r);
    float4 x[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      x[i] = __ldg(reinterpret_cast<const float4*>(p + i * 128 + lane * 4));
      s += (x[i].x + x[i].y) + (x[i].z + x[i].w);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)Cc;
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float a = x[i].x - mean, b = x[i].y - mean, c = x[i].z - mean, d = x[i].w - mean;
      v += (a * a + b * b) + (c * c + d * d);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const float rstd = rsqrtf(v / (float)Cc + eps);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int k = i * 128 + lane * 4;
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma + k));
      const float4 bt = __ldg(reinterpret_cast<const float4*>(beta + k));
      const float4 y = make_float4((x[i].x - mean) * rstd * g.x + bt.x, (x[i].y - mean) * rstd * g.y + bt.y,
                                   (x[i].z - mean) * rstd * g.z + bt.z, (x[i].w - mean) * rstd * g.w + bt.w);
      *reinterpret_cast<float4*>(out + (size_t)r * Cc + k) = y;
    }
  }
}

// LayerNorm backward for the folded prologue: dy = gradient w.r.t. LN(x) (dense [R][Cc], produced by the layer-0 dgrad
// GEMM), x read through the caller's row map, statistics recomputed (cheaper than saving them):
//   xhat = (x - mean) rstd;  g = dy * gamma;  dx = rstd (g - mean(g) - xhat mean(g xhat))
//   dgamma += sum_rows dy xhat;  dbeta += sum_rows dy      (per-CTA partials here, fixed-order reduce below)
// One warp per row, each lane keeps the column partials of its 4*NV columns in registers across its rows.
template <int NV>
__global__ void layernorm_bwd_kernel(const float* __restrict__ x, RowMap x_rows, const float* __restrict__ dy, int R,
                                     int Cc, const float* __restrict__ gamma, float eps, float* __restrict__ dx,
                                     RowMap dx_rows, float* __restrict__ part /* [grid][2][Cc] */,
                                     const int* __restrict__ lengths, int B) {
  extern __shared__ float red[];  // [warps][2][Cc]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  float4 dg[NV], db[NV], gm[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    dg[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    db[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    gm[i] = __ldg(reinterpret_cast<const float4*>(gamma + i * 128 + lane * 4));
  }
  for (int r = blockIdx.x * wpb + warp; r < R; r += gridDim.x * wpb) {
    if (lengths && r / B >= __ldg(lengths + r % B)) {  // padding of a ragged batch: dx = 0, nothing to dgamma / dbeta
      if (dx) {
#pragma unroll
        for (int i = 0; i < NV; ++i)
          *reinterpret_cast<float4*>(dx + dx_rows.off(r) + i * 128 + lane * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      continue;
    }
    const float* px = x + x_rows.off(r);
    const float* pd = dy + (size_t)r * Cc;
    float4 xv[NV], dv[NV];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      xv[i] = __ldg(reinterpret_cast<const float4*>(px + i * 128 + lane * 4));
      dv[i] = *reinterpret_cast<const float4*>(pd + i * 128 + lane * 4);
      s += (xv[i].x + xv[i].y) + (xv[i].z + xv[i].w);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)Cc;
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      xv[i].x -= mean; xv[i].y -= mean; xv[i].z -= mean; xv[i].w -= mean;
      v += (xv[i].x * xv[i].x + xv[i].y * xv[i].y) + (xv[i].z * xv[i].z + xv[i].w * xv[i].w);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const float rstd = rsqrtf(v / (float)Cc + eps);
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      xv[i].x *= rstd; xv[i].y *= rstd; xv[i].z *= rstd; xv[i].w *= rstd;  // xhat
      dg[i].x += dv[i].x * xv[i].x; dg[i].y += dv[i].y * xv[i].y; dg[i].z += dv[i].z * xv[i].z; dg[i].w += dv[i].w * xv[i].w;
      db[i].x += dv[i].x; db[i].y += dv[i].y; db[i].z += dv[i].z; db[i].w += dv[i].w;
      dv[i].x *= gm[i].x; dv[i].y *= gm[i].y; dv[i].z *= gm[i].z; dv[i].w *= gm[i].w;  // g = dy * gamma
      sg += (dv[i].x + dv[i].y) + (dv[i].z + dv[i].w);
      sgx += (dv[i].x * xv[i].x + dv[i].y * xv[i].y) + (dv[i].z * xv[i].z + dv[i].w * xv[i].w);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
      sg += __shfl_xor_sync(0xffffffffu, sg, o);
      sgx += __shfl_xor_sync(0xffffffffu, sgx, o);
    }
    const float mg = sg / (float)Cc, mgx = sgx / (float)Cc;
    if (dx) {
      float* po = dx + dx_rows.off(r);
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        float4 o4;
        o4.x = rstd * (dv[i].x - mg - xv[i].x * mgx);
        o4.y = rstd * (dv[i].y - mg - xv[i].y * mgx);
        o4.z = rstd * (dv[i].z - mg - xv[i].z * mgx);
        o4.w = rstd * (dv[i].w - mg - xv[i].w * mgx);
        *reinterpret_cast<float4*>(po + i * 128 + lane * 4) = o4;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    *reinterpret_cast<float4*>(red + ((size_t)warp * 2 + 0) * Cc + i * 128 + lane * 4) = dg[i];
    *reinterpret_cast<float4*>(red + ((size_t)warp * 2 + 1) * Cc + i * 128 + lane * 4) = db[i];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * Cc; c += blockDim.x) {
    float a = 0.f;
    for (int w2 = 0; w2 < wpb; ++w2) a += red[(size_t)w2 * 2 * Cc + c];  // fixed order
    part[(size_t)blockIdx.x * 2 * Cc + c] = a;
  }
}
__global__ void layernorm_bwd_reduce_kernel(const float* __restrict__ part, int nparts, int Cc, float* __restrict__ dgamma,
                                            float* __restrict__ dbeta, int accumulate) {
  // one warp per column: lane l adds partials l, l+32, ... in order, then a fixed shuffle tree => deterministic, and
  // the ~300 partial rows are read 32 at a time instead of one after the other by a single thread
  const int lane = threadIdx.x & 31, c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (c >= 2 * Cc) return;
  float a = 0.f;
  for (int p2 = lane; p2 < nparts; p2 += 32) a += part[(size_t)p2 * 2 * Cc + c];
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
  if (lane == 0) {
    float* dst = c < Cc ? (dgamma ? dgamma + c : nullptr) : (dbeta ? dbeta + (c - Cc) : nullptr);
    if (dst) *dst = accumulate ? *dst + a : a;
  }
}

// ---- host side -------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encoder() {
  static std::mutex mu;
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  std::lock_guard<std::mutex> lk(mu);
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    else
      cudaGetLastError();
  }
  return fn;
}

// dense row-major [rows, K] fp32 matrix, box = [128 rows, 32 floats], 128-byte swizzle, OOB rows read as zero
bool make_map(CUtensorMap* map, const float* ptr, int rows, int K, long long ld = 0) {
  EncodeTiledFn enc = get_encoder();
  if (!enc) return false;
  if (ld == 0) ld = K;
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)BM};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

// fp16 pairs of W: dense row-major [rows, K] fp16, box = [128 rows, 64 halves] (128-byte rows), 128-byte swizzle
bool make_map16(CUtensorMap* map, const void* ptr, int rows, int K) {
  EncodeTiledFn enc = get_encoder();
  if (!enc || (reinterpret_cast<uintptr_t>(ptr) & 15u) || K % 8 != 0) return false;
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)K * 2};
  cuuint32_t box[2] = {(cuuint32_t)g16::BK, (cuuint32_t)BN};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

// 16-bit A operand read in place through its row map: make_a_f32_map's 3-D map with 2-byte elements and boxes of 64 k
// (128 bytes). TMA only moves the elements, so fp16 and bf16 share the FLOAT16 map type (the zero fill is +0 in both).
bool make_a16_map(CUtensorMap* map, const void* ptr, const RowMap& rows, int M, int K, int* inner) {
  EncodeTiledFn enc = get_encoder();
  if (!enc || (reinterpret_cast<uintptr_t>(ptr) & 15u) || K % 8 != 0) return false;
  const bool dense = rows.inner_n >= M;
  const long long ni = dense ? M : rows.inner_n;
  const long long no = dense ? 1 : (M + ni - 1) / ni;
  const long long si = rows.s_inner, so = dense ? (long long)M * rows.s_inner : rows.s_outer;
  if (!dense && (M % ni != 0 || !(ni % BM == 0 || BM % ni == 0))) return false;
  if (si < K || si % 8 != 0 || so < 1 || so % 8 != 0) return false;
  const cuuint32_t bi = (cuuint32_t)(dense || ni >= BM ? BM : ni);
  cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)ni, (cuuint64_t)no};
  cuuint64_t strides[2] = {(cuuint64_t)si * 2, (cuuint64_t)so * 2};
  cuuint32_t box[3] = {(cuuint32_t)g16::BK, bi, (cuuint32_t)BM / bi};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  *inner = (int)ni;
  return r == CUDA_SUCCESS;
}

// fp32 A operand read in place through its row map: 3-D map {K, inner rows, outer rows} with box {32, bi, 128 / bi},
// so a 128-row tile is one box. Dense rows (inner_n >= M): {K, M, 1}. Rows r = t * B + b of a [T][B] view (tb_rows):
// {K, B, T}, which tiles when B divides 128 or is a multiple of it. Strides must be multiples of 16 bytes.
bool make_a_f32_map(CUtensorMap* map, const float* ptr, const RowMap& rows, int M, int K, int* inner) {
  EncodeTiledFn enc = get_encoder();
  if (!enc || (reinterpret_cast<uintptr_t>(ptr) & 15u) || K % 4 != 0) return false;
  const bool dense = rows.inner_n >= M;
  const long long ni = dense ? M : rows.inner_n;
  const long long no = dense ? 1 : (M + ni - 1) / ni;
  const long long si = rows.s_inner, so = dense ? (long long)M * rows.s_inner : rows.s_outer;
  if (!dense && (M % ni != 0 || !(ni % BM == 0 || BM % ni == 0))) return false;
  if (si < K || si % 4 != 0 || so < 1 || so % 4 != 0) return false;
  const cuuint32_t bi = (cuuint32_t)(dense || ni >= BM ? BM : ni);
  cuuint64_t dims[3] = {(cuuint64_t)K, (cuuint64_t)ni, (cuuint64_t)no};
  cuuint64_t strides[2] = {(cuuint64_t)si * sizeof(float), (cuuint64_t)so * sizeof(float)};
  cuuint32_t box[3] = {(cuuint32_t)BK, bi, (cuuint32_t)BM / bi};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  *inner = (int)ni;
  return r == CUDA_SUCCESS;
}

}  // namespace

size_t gemm_tc_scratch_bytes(int M, int N, int K) { return (size_t)2 * ((size_t)M + N) * K * sizeof(float) + 1024; }

bool gemm_tc_eligible(const GemmParams& p, size_t ws_bytes) {
  if (p.accumulate) return false;
  if (p.M < 1 || p.K < BK || p.K % BK != 0 || p.N % BN != 0) return false;
  if (!p.a_kcontig && p.M % 4 != 0) return false;  // MN-major split copies are dense [K][M]: rows must stay 16-byte aligned
  if (ws_bytes < gemm_tc_scratch_bytes(p.M, p.N, p.K)) return false;
  // the epilogue stores float4 along n
  if ((reinterpret_cast<uintptr_t>(p.C) & 15u) || (p.c_rows.s_outer % 4) || (p.c_rows.s_inner % 4)) return false;
  return get_encoder() != nullptr;
}

int tc_split(const float* src, const RowMap& rows, int R, int Cc, float* hi, float* lo, cudaStream_t stream) {
  const bool vec = (reinterpret_cast<uintptr_t>(src) & 15u) == 0 && rows.s_outer % 4 == 0 && rows.s_inner % 4 == 0;
  size_t nv = (size_t)R * (Cc / 4);
  int blocks = (int)((nv + 255) / 256);
  if (blocks > NUM_SMS * 16) blocks = NUM_SMS * 16;
  if (blocks < 1) blocks = 1;
  ProfScope prof(PROF_MISC, stream);
  split_tf32_kernel<<<blocks, 256, 0, stream>>>(src, rows, R, Cc, hi, lo, vec ? 1 : 0);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

bool tc_a_f32_in_place(const float* A, const RowMap& rows, int M, int K) {
  CUtensorMap m;
  int inner = 0;
  return make_a_f32_map(&m, A, rows, M, K, &inner);
}

int tc_gather_rows(const float* src, const RowMap& rows, int R, int Cc, float* dst, cudaStream_t stream, int* clear,
                   int nclear) {
  const bool vec = (reinterpret_cast<uintptr_t>(src) & 15u) == 0 && rows.s_outer % 4 == 0 && rows.s_inner % 4 == 0;
  if (Cc % 4 != 0) {
    set_error("gather_rows: the row width must be a multiple of 4");
    return B200RNN_ERR_UNSUPPORTED;
  }
  size_t nv = (size_t)R * (Cc / 4);
  int blocks = (int)((nv + 255) / 256);
  if (blocks > NUM_SMS * 16) blocks = NUM_SMS * 16;
  if (blocks < 1) blocks = 1;
  ProfScope prof(PROF_MISC, stream);
  gather_rows_kernel<<<blocks, 256, 0, stream>>>(src, rows, R, Cc, dst, vec ? 1 : 0, clear, clear ? nclear : 0);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

bool tc_available() { return get_encoder() != nullptr; }

float* tc_a_hi(void* ws) { return reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255); }
float* tc_a_lo(void* ws, int M, int K) { return tc_a_hi(ws) + (size_t)M * K; }

int tc_layernorm(const float* src, const RowMap& rows, int R, int Cc, const float* gamma, const float* beta, float eps,
                 float* out, cudaStream_t stream, int* clear, int nclear, const int* lengths, int B) {
  const bool vec = (reinterpret_cast<uintptr_t>(src) & 15u) == 0 && rows.s_outer % 4 == 0 && rows.s_inner % 4 == 0 &&
                   (reinterpret_cast<uintptr_t>(gamma) & 15u) == 0 && (reinterpret_cast<uintptr_t>(beta) & 15u) == 0;
  if (!vec || !(Cc == 128 || Cc == 256 || Cc == 512 || Cc == 1024)) {
    set_error("layernorm: needs 16-byte aligned rows and a feature width of 128, 256, 512 or 1024");
    return B200RNN_ERR_UNSUPPORTED;
  }
  int blocks = (R + 7) / 8;
  if (blocks > NUM_SMS * 8) blocks = NUM_SMS * 8;
  ProfScope prof(PROF_MISC, stream);
  if (!clear) nclear = 0;
#define B200_LNS(NV_) \
  layernorm_kernel<NV_><<<blocks, 256, 0, stream>>>(src, rows, R, Cc, gamma, beta, eps, out, clear, nclear, lengths, B)
  switch (Cc / 128) {  // instantiated widths: 128, 256, 512, 1024 (the reference normalises 256-d audio features)
    case 1: B200_LNS(1); break;
    case 2: B200_LNS(2); break;
    case 4: B200_LNS(4); break;
    default: B200_LNS(8); break;
  }
#undef B200_LNS
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

size_t layernorm_bwd_scratch_floats(int Cc) { return (size_t)LNB_BLOCKS * 2 * Cc; }

int launch_layernorm_bwd(const float* x, const RowMap& x_rows, const float* dy, int R, int Cc, const float* gamma,
                         float eps, float* dx, const RowMap& dx_rows, float* dgamma, float* dbeta, int accumulate,
                         float* part, cudaStream_t stream, const int* lengths, int B) {
  const bool vec = (reinterpret_cast<uintptr_t>(x) & 15u) == 0 && x_rows.s_outer % 4 == 0 && x_rows.s_inner % 4 == 0 &&
                   (reinterpret_cast<uintptr_t>(gamma) & 15u) == 0 && (reinterpret_cast<uintptr_t>(dy) & 15u) == 0 &&
                   (!dx || ((reinterpret_cast<uintptr_t>(dx) & 15u) == 0 && dx_rows.s_outer % 4 == 0 &&
                            dx_rows.s_inner % 4 == 0));
  if (!vec || !(Cc == 128 || Cc == 256 || Cc == 512 || Cc == 1024)) {
    set_error("layernorm_bwd: needs 16-byte aligned rows and a feature width of 128, 256, 512 or 1024");
    return B200RNN_ERR_UNSUPPORTED;
  }
  int blocks = (R + 7) / 8;
  if (blocks > LNB_BLOCKS) blocks = LNB_BLOCKS;
  const size_t smem = (size_t)8 * 2 * Cc * sizeof(float);
  ProfScope prof(PROF_MISC, stream);
  // 8 warps x 2 x Cc floats of per-warp column partials: 64 KB at Cc = 1024, above the 48 KB default limit
  static bool attr[MAX_DEVICES] = {false};
  if (!attr[current_device()]) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(layernorm_bwd_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    attr[current_device()] = true;
  }
#define B200_LNB(NV_) \
  layernorm_bwd_kernel<NV_><<<blocks, 256, smem, stream>>>(x, x_rows, dy, R, Cc, gamma, eps, dx, dx_rows, part, lengths, B)
  switch (Cc / 128) {
    case 1: B200_LNB(1); break;
    case 2: B200_LNB(2); break;
    case 4: B200_LNB(4); break;
    default: B200_LNB(8); break;
  }
#undef B200_LNB
  B200_CUDA_CHECK(cudaGetLastError());
  layernorm_bwd_reduce_kernel<<<(2 * Cc + 7) / 8, 256, 0, stream>>>(part, blocks, Cc, dgamma, dbeta, accumulate);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch(2);
  return B200RNN_OK;
}

namespace {

int num_sms() {
  int sms = NUM_SMS, dev = 0;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

TcArgs tc_args(int M, int N, int K, float* C, const RowMap& c_rows, const float* bias1, const float* bias2,
               int bias2_n, int accumulate, int* ready) {
  TcArgs a;
  memset(&a, 0, sizeof(a));
  a.C = C; a.c_rows = c_rows;
  a.M = M; a.N = N; a.K = K;
  a.bias1 = bias1; a.bias2 = bias2; a.bias2_n = bias2_n;
  a.accumulate = accumulate;
  a.tiles_m = (M + BM - 1) / BM;
  a.tiles_n = N / BN;
  a.splitk = 1;
  a.kb_per_split = (K + BK - 1) / BK;
  a.ready = ready;
  return a;
}

int check_tc_shape(int M, int N, int K, const float* C, const RowMap& c_rows, int* ready, bool splitk,
                   int stream_clusters) {
  if (ready && (splitk || stream_clusters < 1)) {
    set_error("tc_gemm: a streamed launch publishes whole tiles and takes no split-K workspace");
    return B200RNN_ERR_INVALID;
  }
  if (M < 1 || N % BN != 0 || K < 1) {
    set_error("tc_gemm: unsupported shape M=%d N=%d K=%d", M, N, K);
    return B200RNN_ERR_UNSUPPORTED;
  }
  if ((reinterpret_cast<uintptr_t>(C) & 15u) || (c_rows.s_outer % 4) || (c_rows.s_inner % 4)) {
    set_error("tc_gemm: output must be 16-byte aligned with row strides that are multiples of 4 floats");
    return B200RNN_ERR_UNSUPPORTED;
  }
  return B200RNN_OK;
}

// one launch of gemm_tf32x3_kernel over a.tiles_m x a.tiles_n x a.splitk work items (args complete)
int launch_tc(const CUtensorMap (&m)[4], const TcArgs& a, int stream_clusters, cudaStream_t stream) {
  static std::mutex mu;
  static bool attr_done[MAX_DEVICES] = {false};
  {
    const int dev = current_device();
    std::lock_guard<std::mutex> lk(mu);
    if (!attr_done[dev]) {
      B200_CUDA_CHECK(cudaFuncSetAttribute(gemm_tf32x3_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
      B200_CUDA_CHECK(cudaFuncSetAttribute(gemm_tf32x3_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
      B200_CUDA_CHECK(cudaFuncSetAttribute(gemm_tf32x3_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
      B200_CUDA_CHECK(cudaFuncSetAttribute(gemm_tf32x3_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
      B200_CUDA_CHECK(cudaFuncSetAttribute(gemm_f16x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
      B200_CUDA_CHECK(cudaFuncSetAttribute(gemm_n16_kernel<TC_F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
      B200_CUDA_CHECK(cudaFuncSetAttribute(gemm_n16_kernel<TC_BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
      attr_done[dev] = true;
    }
  }
  const int sms = num_sms();
  const int nitems = a.tiles_m * a.tiles_n * a.splitk;
  const bool mn = a.a_mn || a.b_mn;
  auto kernel = a.n16 == TC_BF16 ? gemm_n16_kernel<TC_BF16>
                : a.n16        ? gemm_n16_kernel<TC_F16>
                : a.f16        ? gemm_f16x3_kernel
                : a.tf32 ? (mn ? gemm_tf32x3_kernel<true, true> : gemm_tf32x3_kernel<false, true>)
                         : (mn ? gemm_tf32x3_kernel<true, false> : gemm_tf32x3_kernel<false, false>);
  dim3 grid(nitems < sms ? nitems : sms, 1, 1);
  if (!a.ready) {
    ProfScope prof(PROF_GEMM, stream);
    kernel<<<grid, TC_THREADS, TC_SMEM, stream>>>(m[0], m[1], m[2], m[3], a);
    B200_CUDA_CHECK(cudaGetLastError());
    count_launch();
    return B200RNN_OK;
  }
  // Streamed: 4-CTA clusters (no cluster feature is used). A GPC holds floor(SMs / 4) of them whatever else runs
  // in it, so the GEMM takes exactly `stream_clusters` of the 4-CTA cluster slots and leaves the others to the
  // recurrence's 4-CTA clusters (api.cu); single CTAs spread over the GPCs would fragment them.
  const int want = (nitems + 3) / 4;
  grid.x = 4 * (want < stream_clusters ? want : stream_clusters);
  static const bool debug = getenv("B200RNN_DEBUG") != nullptr;
  if (debug)
    fprintf(stderr, "[b200rnn] streamed x-projection: gemm grid %u (4-CTA clusters) of %d SMs, %d row tiles x %d column tiles\n",
            grid.x, sms, a.tiles_m, a.tiles_n);
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 4;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(TC_THREADS, 1, 1);
  cfg.dynamicSmemBytes = TC_SMEM;
  cfg.stream = stream;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  ProfScope prof(PROF_GEMM, stream);
  B200_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, m[0], m[1], m[2], m[3], a));
  count_launch();
  return B200RNN_OK;
}

}  // namespace

void tc_splitk_plan(int M, int N, int K, bool have_ws, size_t ws_bytes, int* splitk_out, int* kb_per_split) {
  const int ntiles = ((M + BM - 1) / BM) * (N / BN);
  const int nkb = (K + BK - 1) / BK;
  const int sms = num_sms();
  // split-K when the tile count cannot fill the chip and K is long (the wgrad shapes: K = T*B)
  int splitk = 1;
  if (have_ws && ntiles * 2 <= sms && nkb >= 16) {
    splitk = sms / ntiles;
    if (splitk > nkb / 8) splitk = nkb / 8;
    const size_t per = (size_t)M * N * sizeof(float);
    while (splitk > 1 && per * splitk > ws_bytes) --splitk;
    if (splitk < 1) splitk = 1;
  }
  *kb_per_split = (nkb + splitk - 1) / splitk;
  *splitk_out = (nkb + *kb_per_split - 1) / *kb_per_split;
}

// C[M,N] (+)= A[M,K] * B[N,K]^T (+ biases), operands already split into hi/lo matrices (K- or MN-major).
int tc_gemm_presplit(const TcOperand& A, const TcOperand& B, int M, int N, int K, float* C, const RowMap& c_rows,
                     const float* bias1, const float* bias2, int bias2_n, int accumulate, void* splitk_ws,
                     size_t splitk_ws_bytes, cudaStream_t stream, int* ready, int stream_clusters, bool tf32) {
  int rc = check_tc_shape(M, N, K, C, c_rows, ready, splitk_ws != nullptr, stream_clusters);
  if (rc) return rc;
  // MN-major operands are read by the kernel's own loads: their tensor maps stay zero and unused
  CUtensorMap m[4] = {};
  const bool ok_a = A.mn || (make_map(&m[0], A.hi, M, K, A.ld) && (tf32 || make_map(&m[1], A.lo, M, K, A.ld)));
  const bool ok_b = B.mn || (make_map(&m[2], B.hi, N, K, B.ld) && (tf32 || make_map(&m[3], B.lo, N, K, B.ld)));
  if (!ok_a || !ok_b) {
    set_error("tc_gemm: cuTensorMapEncodeTiled failed (operands must be 16-byte aligned, ld %% 4 == 0)");
    return B200RNN_ERR_CUDA;
  }
  TcArgs a = tc_args(M, N, K, C, c_rows, bias1, bias2, bias2_n, accumulate, ready);
  a.a_mn = A.mn ? 1 : 0;
  a.b_mn = B.mn ? 1 : 0;
  a.a_hi = A.hi; a.a_lo = A.lo; a.lda = A.ld;
  a.b_hi = B.hi; a.b_lo = B.lo; a.ldb = B.ld;
  a.tf32 = tf32 ? 1 : 0;
  tc_splitk_plan(M, N, K, splitk_ws != nullptr, splitk_ws_bytes, &a.splitk, &a.kb_per_split);
  a.partial = static_cast<float*>(splitk_ws);
  rc = launch_tc(m, a, stream_clusters, stream);
  if (rc) return rc;
  if (a.splitk > 1)
    return launch_splitk_reduce(a.partial, a.splitk, M, N, C, c_rows, bias1, bias2, bias2_n, accumulate, stream);
  return B200RNN_OK;
}

// C[M,N] = A[M,K] * B[N,K]^T + biases with A in fp32, read in place through its row map and split on chip; B K-major
// presplit. Same operands, same MMAs, same sums as tc_gemm_presplit on split(A), so C is bit-identical.
int tc_gemm_f32a(const float* A, const RowMap& a_rows, const TcOperand& B, int M, int N, int K, float* C,
                 const RowMap& c_rows, const float* bias1, const float* bias2, int bias2_n, cudaStream_t stream,
                 int* ready, int stream_clusters, bool tf32) {
  int rc = check_tc_shape(M, N, K, C, c_rows, ready, false, stream_clusters);
  if (rc) return rc;
  if (B.mn || K % BK != 0) {
    set_error("tc_gemm: the fp32-A path takes a K-major presplit B and K %% 32 == 0");
    return B200RNN_ERR_UNSUPPORTED;
  }
  CUtensorMap m[4] = {};
  int inner = 0;
  if (!make_a_f32_map(&m[0], A, a_rows, M, K, &inner)) {
    set_error("tc_gemm: the fp32 A operand cannot be read in place (16-byte aligned rows; batch dividing 128 or a "
              "multiple of it)");
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (!make_map(&m[2], B.hi, N, K, B.ld) || (!tf32 && !make_map(&m[3], B.lo, N, K, B.ld))) {
    set_error("tc_gemm: cuTensorMapEncodeTiled failed (operands must be 16-byte aligned, ld %% 4 == 0)");
    return B200RNN_ERR_CUDA;
  }
  TcArgs a = tc_args(M, N, K, C, c_rows, bias1, bias2, bias2_n, 0, ready);
  a.a_f32 = 1;
  a.a_inner = inner;
  a.tf32 = tf32 ? 1 : 0;
  return launch_tc(m, a, stream_clusters, stream);
}

int tc_split_w16(const float* W, const RowMap& rows, int N, int K, void* w16, cudaStream_t stream) {
  if (!g16::shape_ok(N, K) || !w16 || (reinterpret_cast<uintptr_t>(w16) % g16::ALIGN)) {
    set_error("split_w16: needs N %% 128 == 0, K %% 64 == 0 and a 256-byte aligned destination (N=%d K=%d)", N, K);
    return B200RNN_ERR_UNSUPPORTED;
  }
  const g16::W16 l = g16::w16_layout(N, K);
  unsigned char* b = static_cast<unsigned char*>(w16);
  int blocks = (N + 7) / 8;
  if (blocks > NUM_SMS * 4) blocks = NUM_SMS * 4;
  ProfScope prof(PROF_MISC, stream);
  split_w16_kernel<<<blocks, 256, 0, stream>>>(W, rows, N, K, reinterpret_cast<__half*>(b + l.hi),
                                               reinterpret_cast<__half*>(b + l.lo), reinterpret_cast<int*>(b + l.exp));
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

// C[M,N] = A[M,K] * W[N,K]^T + biases with A in fp32, read in place and split into fp16 pairs on chip; W as fp16 pairs
// at w16 (tc_split_w16). A tile's result depends on its operands only, not on the grid or on streaming.
int tc_gemm_f16a(const float* A, const RowMap& a_rows, const void* w16, int M, int N, int K, float* C,
                 const RowMap& c_rows, const float* bias1, const float* bias2, int bias2_n, cudaStream_t stream,
                 int* ready, int stream_clusters) {
  int rc = check_tc_shape(M, N, K, C, c_rows, ready, false, stream_clusters);
  if (rc) return rc;
  if (!g16::shape_ok(N, K)) {
    set_error("tc_gemm: the fp16-pair path takes N %% 128 == 0 and K %% 64 == 0 (N=%d K=%d)", N, K);
    return B200RNN_ERR_UNSUPPORTED;
  }
  CUtensorMap m[4] = {};
  int inner = 0;
  if (!make_a_f32_map(&m[0], A, a_rows, M, K, &inner)) {
    set_error("tc_gemm: the fp32 A operand cannot be read in place (16-byte aligned rows; batch dividing 128 or a "
              "multiple of it)");
    return B200RNN_ERR_UNSUPPORTED;
  }
  const g16::W16 l = g16::w16_layout(N, K);
  const unsigned char* b = static_cast<const unsigned char*>(w16);
  if (!make_map16(&m[2], b + l.hi, N, K) || !make_map16(&m[3], b + l.lo, N, K)) {
    set_error("tc_gemm: cuTensorMapEncodeTiled failed for the fp16 weight pairs");
    return B200RNN_ERR_CUDA;
  }
  TcArgs a = tc_args(M, N, K, C, c_rows, bias1, bias2, bias2_n, 0, ready);
  a.a_f32 = 1;
  a.a_inner = inner;
  a.kb_per_split = K / g16::BK;
  a.w_exp = reinterpret_cast<const int*>(b + l.exp);
  a.f16 = 1;
  return launch_tc(m, a, stream_clusters, stream);
}

int launch_gemm_tc(const GemmParams& p, void* ws, size_t ws_bytes, cudaStream_t stream) {
  if (!gemm_tc_eligible(p, ws_bytes)) {
    set_error("gemm_tc: problem not eligible for the tensor-core path");
    return B200RNN_ERR_UNSUPPORTED;
  }
  const bool tf32 = p.tc_tf32 != 0;
  float* a_hi = tc_a_hi(ws);
  float* a_lo = tc_a_lo(ws, p.M, p.K);
  const float* b_hi = p.tc_b_hi;
  const float* b_lo = p.tc_b_lo;
  int rc = B200RNN_OK;
  // a_kcontig: A is [M rows][K]; else A is [K rows][M] (MN-major): the split copy keeps the source's orientation
  if (!p.tc_a_f32)
    rc = p.a_kcontig ? tc_split(p.A, p.a_rows, p.M, p.K, a_hi, tf32 ? nullptr : a_lo, stream)
                     : tc_split(p.A, p.a_rows, p.K, p.M, a_hi, tf32 ? nullptr : a_lo, stream);
  if (rc) return rc;
  static const bool debug = getenv("B200RNN_DEBUG") != nullptr;
  // fp16 pairs (the no-grad forward of b200rnn_forward_fused): W as split by b200rnn_prepare_weights, else split here
  // into the room of the TF32 W split; a shape it does not take runs the 3xTF32 fp32-A kernel
  const bool h16 = p.tc_h16 && p.tc_a_f32 && p.b_kcontig && !tf32 && g16::shape_ok(p.N, p.K);
  if (debug && p.tc_a_f32)
    fprintf(stderr, "[b200rnn] forward x-projection: M=%d N=%d K=%d math=%s weights=%s a=%s\n", p.M, p.N, p.K,
            h16 ? "f16x3" : tf32 ? "tf32" : "3xtf32",
            (h16 ? p.tc_b_h16 != nullptr : b_hi != nullptr) ? "cached" : "split", p.a_route ? p.a_route : "tma");
  if (h16) {
    const void* w16 = p.tc_b_h16;
    if (!w16) {
      void* dst = a_lo + (size_t)p.M * p.K;
      rc = tc_split_w16(p.B, p.b_rows, p.N, p.K, dst, stream);
      if (rc) return rc;
      w16 = dst;
    }
    return tc_gemm_f16a(p.A, p.a_rows, w16, p.M, p.N, p.K, p.C, p.c_rows, p.bias1, p.bias2, p.bias2_n, stream,
                        p.tc_ready, p.tc_stream_clusters);
  }
  if (!b_hi || (!b_lo && !tf32)) {  // single-pass TF32 reads and writes only hi
    float* w_hi = a_lo + (size_t)p.M * p.K;
    float* w_lo = tf32 ? nullptr : w_hi + (size_t)p.N * p.K;
    rc = p.b_kcontig ? tc_split(p.B, p.b_rows, p.N, p.K, w_hi, w_lo, stream)
                     : tc_split(p.B, p.b_rows, p.K, p.N, w_hi, w_lo, stream);
    if (rc) return rc;
    b_hi = w_hi;
    b_lo = w_lo;
  }
  TcOperand B{b_hi, b_lo, p.b_kcontig ? p.K : p.N, !p.b_kcontig};
  if (p.tc_a_f32)
    return tc_gemm_f32a(p.A, p.a_rows, B, p.M, p.N, p.K, p.C, p.c_rows, p.bias1, p.bias2, p.bias2_n, stream,
                        p.tc_ready, p.tc_stream_clusters, tf32);
  TcOperand A{a_hi, a_lo, p.a_kcontig ? p.K : p.M, !p.a_kcontig};
  return tc_gemm_presplit(A, B, p.M, p.N, p.K, p.C, p.c_rows, p.bias1, p.bias2, p.bias2_n, 0, nullptr, 0, stream,
                          p.tc_ready, p.tc_stream_clusters, tf32);
}

bool tc_gemm_n16_ok(const void* A, const RowMap& a_rows, const void* W, int M, int N, int K) {
  CUtensorMap m;
  int inner = 0;
  return M >= 1 && N % BN == 0 && N > 0 && K % 8 == 0 && K > 0 && (reinterpret_cast<uintptr_t>(W) & 15u) == 0 &&
         make_a16_map(&m, A, a_rows, M, K, &inner);
}

int tc_gemm_n16(const void* A, const RowMap& a_rows, const void* W, int M, int N, int K, int dt, float* C,
                const RowMap& c_rows, const float* bias1, const float* bias2, int bias2_n, cudaStream_t stream,
                const char* a_route) {
  int rc = check_tc_shape(M, N, K, C, c_rows, nullptr, false, 0);
  if (rc) return rc;
  CUtensorMap m[4] = {};
  int inner = 0;
  if (!make_a16_map(&m[0], A, a_rows, M, K, &inner) || !make_map16(&m[2], W, N, K)) {
    set_error("tc_gemm: the 16-bit operands cannot be read by TMA (16-byte aligned rows, K %% 8 == 0, batch dividing "
              "128 or a multiple of it)");
    return B200RNN_ERR_UNSUPPORTED;
  }
  static const bool debug = getenv("B200RNN_DEBUG") != nullptr;
  if (debug)
    fprintf(stderr, "[b200rnn] forward x-projection: M=%d N=%d K=%d math=%s weights=native a=%s\n", M, N, K,
            dt == DT_BF16 ? "bf16" : "f16", a_route ? a_route : "tma");
  TcArgs a = tc_args(M, N, K, C, c_rows, bias1, bias2, bias2_n, 0, nullptr);
  a.a_f32 = 1;  // one thread issues the A and W boxes
  a.a_inner = inner;
  a.kb_per_split = (K + g16::BK - 1) / g16::BK;
  a.n16 = dt == DT_BF16 ? TC_BF16 : TC_F16;
  return launch_tc(m, a, 0, stream);
}

}  // namespace b200rnn
