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
//   warpgroups 1-2: consumers — 64 rows of the tile each: wgmma.m64n128k8.tf32 from shared-memory descriptors,
//                   12 per stage, then the round-to-nearest flush and finally the epilogue (+ folded biases).
#include <cuda.h>  // CUtensorMap types only; the encoder is fetched through cudaGetDriverEntryPoint
#include <mutex>

#include "gemm_f32.cuh"
#include "profile.cuh"
#include "ptx.cuh"

namespace b200rnn {

namespace {

constexpr int BM = 128, BN = 128, BK = 32, STAGES = 3;
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
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// raise the expected transaction bytes of the current phase without arriving
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.expect_tx.relaxed.cta.shared::cta.b64 [%0], %1;" ::"r"(ptx::smem_u32(bar)), "r"(bytes)
               : "memory");
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
};

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

// Persistent: each CTA walks work items blockIdx.x, +gridDim.x, ... (m fastest, so consecutive tiles of a CTA mostly
// share their W tile rows in L2). Producer and consumers loop independently over the same item sequence and meet only
// through the full / empty mbarriers of the shared-memory ring.
__global__ void __launch_bounds__(TC_THREADS, 1)
    gemm_tf32x3_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                       const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
                       const TcArgs args) {
  extern __shared__ unsigned char smem_raw[];
  // aligned by offset so that the compiler keeps the shared state space (LDS/STS instead of generic LD/ST)
  unsigned char* base = smem_raw + ((1024u - (ptx::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(base + STAGES * STAGE_BYTES);
  uint64_t* empty = full + STAGES;

  // canonical warp index: the shuffle makes it warp-uniform for the compiler, so the single-thread TMA issue stays on
  // the uniform datapath (no per-instruction R2UR broadcast loop around UTMALDG)
  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int nkb_total = (args.K + BK - 1) / BK;  // the K tail reads as zero
  const int ntiles = args.tiles_m * args.tiles_n;
  const int nitems = ntiles * args.splitk;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(&full[s], 128);  // every producer thread, after its own stores
      ptx::mbar_init(&empty[s], 8);   // one arrival per consumer warp
    }
    ptx::fence_mbar_init();
    if (!args.a_mn) {
      prefetch_tmap(&map_a_hi);
      prefetch_tmap(&map_a_lo);
    }
    if (!args.b_mn) {
      prefetch_tmap(&map_b_hi);
      prefetch_tmap(&map_b_lo);
    }
  }
  __syncthreads();

  if (warp < 4) {
    const int t = threadIdx.x;
    const uint32_t tx = (args.a_mn ? 0u : 2u * TILE_BYTES) + (args.b_mn ? 0u : 2u * TILE_BYTES);
    int it = 0;  // running k-block counter across items (ring position)
    for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
      const int tile = item % ntiles, ks = item / ntiles;
      const int m0 = (tile % args.tiles_m) * BM, n0 = (tile / args.tiles_m) * BN;
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
            if (!args.a_mn) {
              tma_load_2d(st + 0 * TILE_BYTES, &map_a_hi, kb * BK, m0, &full[s]);
              tma_load_2d(st + 1 * TILE_BYTES, &map_a_lo, kb * BK, m0, &full[s]);
            }
            if (!args.b_mn) {
              tma_load_2d(st + 2 * TILE_BYTES, &map_b_hi, kb * BK, n0, &full[s]);
              tma_load_2d(st + 3 * TILE_BYTES, &map_b_lo, kb * BK, n0, &full[s]);
            }
          }
          __syncwarp();
        }
        if (args.a_mn) {
          load_mn_tile(st + 0 * TILE_BYTES, args.a_hi, args.lda, args.M, args.K, m0, kb * BK, t);
          load_mn_tile(st + 1 * TILE_BYTES, args.a_lo, args.lda, args.M, args.K, m0, kb * BK, t);
        }
        if (args.b_mn) {
          load_mn_tile(st + 2 * TILE_BYTES, args.b_hi, args.ldb, args.N, args.K, n0, kb * BK, t);
          load_mn_tile(st + 3 * TILE_BYTES, args.b_lo, args.ldb, args.N, args.K, n0, kb * BK, t);
        }
        if (args.a_mn || args.b_mn) ptx::fence_proxy_async();  // generic stores -> visible to wgmma (async proxy)
        ptx::mbar_arrive(&full[s]);
      }
    }
  } else {
    const int wg = (threadIdx.x >> 7) - 1;   // consumer warpgroup: tile rows [64 wg, 64 wg + 64)
    const int wq = warp & 3;                 // warp within the warpgroup: 16 accumulator rows each
    int it = 0;
    for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
      const int tile = item % ntiles, ks = item / ntiles;
      const int nkb = min(nkb_total, (ks + 1) * args.kb_per_split) - ks * args.kb_per_split;
      const int m0 = (tile % args.tiles_m) * BM, n0 = (tile / args.tiles_m) * BN;
      float total[64], acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) total[i] = 0.f;
      for (int kb = 0; kb < nkb; ++kb, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (it / STAGES) & 1;
        ptx::mbar_wait(&full[s], ph);
        const uint32_t st = ptx::smem_u32(base + s * STAGE_BYTES);
        const uint64_t a_hi = make_kmajor_sw128_desc(st + 0 * TILE_BYTES + wg * 8192);
        const uint64_t a_lo = make_kmajor_sw128_desc(st + 1 * TILE_BYTES + wg * 8192);
        const uint64_t b_hi = make_kmajor_sw128_desc(st + 2 * TILE_BYTES);
        const uint64_t b_lo = make_kmajor_sw128_desc(st + 3 * TILE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 8; ++k) {
          const uint64_t adv = (uint64_t)(k * (32 >> 4));  // K step of 8 tf32 = 32 bytes inside the swizzle atom
          wgmma_tf32_m64n128k8(acc, a_lo + adv, b_hi + adv, k != 0);
          wgmma_tf32_m64n128k8(acc, a_hi + adv, b_lo + adv, 1);
          wgmma_tf32_m64n128k8(acc, a_hi + adv, b_hi + adv, 1);
        }
        wgmma_commit();
        wgmma_wait0();
        reg_fence(acc);
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&empty[s]);  // this warp's share of the stage has been read
#pragma unroll
        for (int i = 0; i < 64; ++i) total[i] += acc[i];
      }
      // accumulator fragment: element i sits at row 16 wq + lane/4 + 8 ((i/2) & 1), column 8 (i/4) + 2 (lane%4) + i%2
      const int r0 = m0 + wg * 64 + wq * 16 + (lane >> 2);
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
          if (args.splitk == 1) {
            const int n = n0 + col;
            if (args.bias1) { o.x += __ldg(args.bias1 + n); o.y += __ldg(args.bias1 + n + 1); }
            if (args.bias2) {
              if (n < args.bias2_n) o.x += __ldg(args.bias2 + n);
              if (n + 1 < args.bias2_n) o.y += __ldg(args.bias2 + n + 1);
            }
            if (args.accumulate) {
              const float2 old = *reinterpret_cast<const float2*>(crow + col);
              o.x += old.x; o.y += old.y;
            }
          }
          *reinterpret_cast<float2*>(crow + col) = o;
        }
      }
    }
  }
}

// x = hi + lo with hi = round-to-nearest TF32 (kept in a 32-bit container), lo = x - hi (exact in fp32).
// Reads rows through a RowMap (batch_first / permuted inputs), writes two dense [M,K] matrices.
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
    *reinterpret_cast<float4*>(lo + (size_t)m * K + k) = l;
  }
}

// LayerNorm(row) * gamma + beta, then the TF32 split — the prologue of audio_gru_whole.py:104 / fuse_net_whole.py:360
// folded into the operand preparation of K1 (SURVEY.md 8f rank 1). One warp per row; Cc % 128 == 0, Cc <= 1024.
template <int NV>  // float4 per lane
__global__ void layernorm_split_kernel(const float* __restrict__ src, RowMap rows, int R, int Cc,
                                       const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                       float* __restrict__ hi, float* __restrict__ lo, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < R; r += gridDim.x * wpb) {
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
      float y[4] = {(x[i].x - mean) * rstd * g.x + bt.x, (x[i].y - mean) * rstd * g.y + bt.y,
                    (x[i].z - mean) * rstd * g.z + bt.z, (x[i].w - mean) * rstd * g.w + bt.w};
      float h[4], l[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        uint32_t t;
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(y[e]));
        h[e] = __uint_as_float(t);
        l[e] = y[e] - h[e];
      }
      *reinterpret_cast<float4*>(hi + (size_t)r * Cc + k) = make_float4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<float4*>(lo + (size_t)r * Cc + k) = make_float4(l[0], l[1], l[2], l[3]);
      if (out) *reinterpret_cast<float4*>(out + (size_t)r * Cc + k) = make_float4(y[0], y[1], y[2], y[3]);  // for backward
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
                                     RowMap dx_rows, float* __restrict__ part /* [grid][2][Cc] */) {
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

bool tc_disabled() {
  static const bool off = getenv("B200RNN_NO_TC") != nullptr;
  return off;
}

}  // namespace

size_t gemm_tc_scratch_bytes(int M, int N, int K) { return (size_t)2 * ((size_t)M + N) * K * sizeof(float) + 1024; }

bool gemm_tc_eligible(const GemmParams& p, size_t ws_bytes) {
  if (tc_disabled()) return false;
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

bool tc_available() { return !tc_disabled() && get_encoder() != nullptr; }

float* tc_a_hi(void* ws) { return reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255); }
float* tc_a_lo(void* ws, int M, int K) { return tc_a_hi(ws) + (size_t)M * K; }

int tc_layernorm_split(const float* src, const RowMap& rows, int R, int Cc, const float* gamma, const float* beta,
                       float eps, float* hi, float* lo, cudaStream_t stream, float* out) {
  const bool vec = (reinterpret_cast<uintptr_t>(src) & 15u) == 0 && rows.s_outer % 4 == 0 && rows.s_inner % 4 == 0 &&
                   (reinterpret_cast<uintptr_t>(gamma) & 15u) == 0 && (reinterpret_cast<uintptr_t>(beta) & 15u) == 0;
  if (!vec || !(Cc == 128 || Cc == 256 || Cc == 512 || Cc == 1024)) {
    set_error("layernorm_split: needs 16-byte aligned rows and a feature width of 128, 256, 512 or 1024");
    return B200RNN_ERR_UNSUPPORTED;
  }
  int blocks = (R + 7) / 8;
  if (blocks > NUM_SMS * 8) blocks = NUM_SMS * 8;
  ProfScope prof(PROF_MISC, stream);
  switch (Cc / 128) {  // instantiated widths: 128, 256, 512, 1024 (the reference normalises 256-d audio features)
    case 1: layernorm_split_kernel<1><<<blocks, 256, 0, stream>>>(src, rows, R, Cc, gamma, beta, eps, hi, lo, out); break;
    case 2: layernorm_split_kernel<2><<<blocks, 256, 0, stream>>>(src, rows, R, Cc, gamma, beta, eps, hi, lo, out); break;
    case 4: layernorm_split_kernel<4><<<blocks, 256, 0, stream>>>(src, rows, R, Cc, gamma, beta, eps, hi, lo, out); break;
    default: layernorm_split_kernel<8><<<blocks, 256, 0, stream>>>(src, rows, R, Cc, gamma, beta, eps, hi, lo, out); break;
  }
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

size_t layernorm_bwd_scratch_floats(int Cc) { return (size_t)LNB_BLOCKS * 2 * Cc; }

int launch_layernorm_bwd(const float* x, const RowMap& x_rows, const float* dy, int R, int Cc, const float* gamma,
                         float eps, float* dx, const RowMap& dx_rows, float* dgamma, float* dbeta, int accumulate,
                         float* part, cudaStream_t stream) {
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
  layernorm_bwd_kernel<NV_><<<blocks, 256, smem, stream>>>(x, x_rows, dy, R, Cc, gamma, eps, dx, dx_rows, part)
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

// C[M,N] (+)= A[M,K] * B[N,K]^T (+ biases), operands already split into hi/lo matrices (K- or MN-major).
int tc_gemm_presplit(const TcOperand& A, const TcOperand& B, int M, int N, int K, float* C, const RowMap& c_rows,
                     const float* bias1, const float* bias2, int bias2_n, int accumulate, void* splitk_ws,
                     size_t splitk_ws_bytes, cudaStream_t stream) {
  if (M < 1 || N % BN != 0 || K < 1) {
    set_error("tc_gemm: unsupported shape M=%d N=%d K=%d", M, N, K);
    return B200RNN_ERR_UNSUPPORTED;
  }
  if ((reinterpret_cast<uintptr_t>(C) & 15u) || (c_rows.s_outer % 4) || (c_rows.s_inner % 4)) {
    set_error("tc_gemm: output must be 16-byte aligned with row strides that are multiples of 4 floats");
    return B200RNN_ERR_UNSUPPORTED;
  }
  // MN-major operands are read by the kernel's own loads: their tensor maps stay zero and unused
  CUtensorMap m_ahi{}, m_alo{}, m_bhi{}, m_blo{};
  const bool ok_a = A.mn || (make_map(&m_ahi, A.hi, M, K, A.ld) && make_map(&m_alo, A.lo, M, K, A.ld));
  const bool ok_b = B.mn || (make_map(&m_bhi, B.hi, N, K, B.ld) && make_map(&m_blo, B.lo, N, K, B.ld));
  if (!ok_a || !ok_b) {
    set_error("tc_gemm: cuTensorMapEncodeTiled failed (operands must be 16-byte aligned, ld %% 4 == 0)");
    return B200RNN_ERR_CUDA;
  }
  static std::mutex mu;
  static bool attr_done[MAX_DEVICES] = {false};
  {
    const int dev = current_device();
    std::lock_guard<std::mutex> lk(mu);
    if (!attr_done[dev]) {
      B200_CUDA_CHECK(cudaFuncSetAttribute(gemm_tf32x3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM));
      attr_done[dev] = true;
    }
  }
  int sms = NUM_SMS;
  {
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  TcArgs a;
  a.C = C; a.c_rows = c_rows;
  a.M = M; a.N = N; a.K = K;
  a.bias1 = bias1; a.bias2 = bias2; a.bias2_n = bias2_n;
  a.accumulate = accumulate;
  a.a_mn = A.mn ? 1 : 0;
  a.b_mn = B.mn ? 1 : 0;
  a.a_hi = A.hi; a.a_lo = A.lo; a.lda = A.ld;
  a.b_hi = B.hi; a.b_lo = B.lo; a.ldb = B.ld;
  a.tiles_m = (M + BM - 1) / BM;
  a.tiles_n = N / BN;
  const int ntiles = a.tiles_m * a.tiles_n;
  const int nkb = (K + BK - 1) / BK;
  // split-K when the tile count cannot fill the chip and K is long (the wgrad shapes: K = T*B)
  int splitk = 1;
  if (splitk_ws && ntiles * 2 <= sms && nkb >= 16) {
    splitk = sms / ntiles;
    if (splitk > nkb / 8) splitk = nkb / 8;
    const size_t per = (size_t)M * N * sizeof(float);
    while (splitk > 1 && per * splitk > splitk_ws_bytes) --splitk;
    if (splitk < 1) splitk = 1;
  }
  a.kb_per_split = (nkb + splitk - 1) / splitk;
  a.splitk = (nkb + a.kb_per_split - 1) / a.kb_per_split;
  a.partial = static_cast<float*>(splitk_ws);
  const int nitems = ntiles * a.splitk;
  dim3 grid(nitems < sms ? nitems : sms, 1, 1);
  {
    ProfScope prof(PROF_GEMM, stream);
    gemm_tf32x3_kernel<<<grid, TC_THREADS, TC_SMEM, stream>>>(m_ahi, m_alo, m_bhi, m_blo, a);
    B200_CUDA_CHECK(cudaGetLastError());
    count_launch();
  }
  if (a.splitk > 1)
    return launch_splitk_reduce(a.partial, a.splitk, M, N, C, c_rows, bias1, bias2, bias2_n, accumulate, stream);
  return B200RNN_OK;
}

int launch_gemm_tc(const GemmParams& p, void* ws, size_t ws_bytes, cudaStream_t stream) {
  if (!gemm_tc_eligible(p, ws_bytes)) {
    set_error("gemm_tc: problem not eligible for the tensor-core path");
    return B200RNN_ERR_UNSUPPORTED;
  }
  float* a_hi = tc_a_hi(ws);
  float* a_lo = tc_a_lo(ws, p.M, p.K);
  const float* b_hi = p.tc_b_hi;
  const float* b_lo = p.tc_b_lo;
  int rc = B200RNN_OK;
  // a_kcontig: A is [M rows][K]; else A is [K rows][M] (MN-major): the split copy keeps the source's orientation
  if (!p.tc_a_presplit)
    rc = p.a_kcontig ? tc_split(p.A, p.a_rows, p.M, p.K, a_hi, a_lo, stream)
                     : tc_split(p.A, p.a_rows, p.K, p.M, a_hi, a_lo, stream);
  if (rc) return rc;
  if (!b_hi || !b_lo) {
    float* w_hi = a_lo + (size_t)p.M * p.K;
    float* w_lo = w_hi + (size_t)p.N * p.K;
    rc = p.b_kcontig ? tc_split(p.B, p.b_rows, p.N, p.K, w_hi, w_lo, stream)
                     : tc_split(p.B, p.b_rows, p.K, p.N, w_hi, w_lo, stream);
    if (rc) return rc;
    b_hi = w_hi;
    b_lo = w_lo;
  }
  TcOperand A{a_hi, a_lo, p.a_kcontig ? p.K : p.M, !p.a_kcontig}, B{b_hi, b_lo, p.b_kcontig ? p.K : p.N, !p.b_kcontig};
  return tc_gemm_presplit(A, B, p.M, p.N, p.K, p.C, p.c_rows, p.bias1, p.bias2, p.bias2_n, 0, nullptr, 0, stream);
}

}  // namespace b200rnn
