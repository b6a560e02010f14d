// gemm_f32.cu — fp32 FFMA tile GEMM for the time-parallel parts of the path:
//   K1  Gi   = X   * W_ih^T + b          (A k-contig, B k-contig)
//   K6  dX   = dGi * W_ih                (A k-contig, B n-contig)
//       dW   = dGi^T * X  (split-K)      (A m-contig, B n-contig)
// Rows may be two-level strided (RowMap) so batch_first / permuted inputs are read in place.
// fp32 FFMA on purpose: the reference path is fp32 (torch rnn.py:1221-1224, :842-847) and parity is
// judged at 1e-5; the dense shapes go to the 3xTF32 tensor-core kernel (gemm_tc.cu), this one takes the rest.
#include <stdlib.h>
#include <string.h>

#include "gemm_f32.cuh"
#include "profile.cuh"

namespace b200rnn {

namespace {

constexpr int BK = 16;
constexpr int NTHREADS = 256;

struct GemmDev {
  const float* A;
  RowMap a_rows;
  const float* B;
  RowMap b_rows;
  float* C;
  RowMap c_rows;
  int M, N, K;
  const float* bias1;
  const float* bias2;
  int bias2_n;
  int accumulate;
  int a_vec, b_vec;  // float4 global loads legal (base + strides 16B aligned)
  int splitk;        // >1: write partial[z][M][N]
  int k_chunk;       // K range per z (multiple of BK)
  float* partial;
};

// Load a (ROWS x BK) operand tile into registers; KC: rows indexed by the non-k dim, k contiguous.
template <bool KC, int BMN>
__device__ __forceinline__ void load_tile(const float* __restrict__ base, const RowMap& rows, int vec_ok,
                                          int mn0, int MN, int k0, int kend, float4 (&reg)[BMN / 64]) {
#pragma unroll
  for (int j = 0; j < BMN / 64; ++j) {
    int f = threadIdx.x + j * NTHREADS;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (KC) {
      int row = f >> 2, kq = (f & 3) * 4;
      int mn = mn0 + row, k = k0 + kq;
      if (mn < MN && k < kend) {
        const float* p = base + rows.off(mn) + k;
        if (vec_ok && k + 3 < kend) {
          v = __ldg(reinterpret_cast<const float4*>(p));
        } else {
          v.x = __ldg(p);
          if (k + 1 < kend) v.y = __ldg(p + 1);
          if (k + 2 < kend) v.z = __ldg(p + 2);
          if (k + 3 < kend) v.w = __ldg(p + 3);
        }
      }
    } else {
      int krow = f / (BMN / 4), mq = (f % (BMN / 4)) * 4;
      int k = k0 + krow, mn = mn0 + mq;
      if (k < kend && mn < MN) {
        const float* p = base + rows.off(k) + mn;
        if (vec_ok && mn + 3 < MN) {
          v = __ldg(reinterpret_cast<const float4*>(p));
        } else {
          v.x = __ldg(p);
          if (mn + 1 < MN) v.y = __ldg(p + 1);
          if (mn + 2 < MN) v.z = __ldg(p + 2);
          if (mn + 3 < MN) v.w = __ldg(p + 3);
        }
      }
    }
    reg[j] = v;
  }
}

// Store the register tile to shared memory as S[k][mn] (leading dim BMN+4).
template <bool KC, int BMN>
__device__ __forceinline__ void store_tile(float* __restrict__ S, const float4 (&reg)[BMN / 64]) {
  constexpr int LD = BMN + 4;
#pragma unroll
  for (int j = 0; j < BMN / 64; ++j) {
    int f = threadIdx.x + j * NTHREADS;
    if (KC) {
      int row = f >> 2, kq = (f & 3) * 4;
      S[(kq + 0) * LD + row] = reg[j].x;
      S[(kq + 1) * LD + row] = reg[j].y;
      S[(kq + 2) * LD + row] = reg[j].z;
      S[(kq + 3) * LD + row] = reg[j].w;
    } else {
      int krow = f / (BMN / 4), mq = (f % (BMN / 4)) * 4;
      *reinterpret_cast<float4*>(&S[krow * LD + mq]) = reg[j];
    }
  }
}

template <bool A_KC, bool B_KC, int BM, int BN>
__global__ void __launch_bounds__(NTHREADS) gemm_f32_kernel(const GemmDev p) {
  constexpr int TM = BM / 16, TN = BN / 16;  // per-thread micro tile (4 or 8)
  constexpr int LDA = BM + 4, LDB = BN + 4;
  __shared__ __align__(16) float As[2][BK * LDA];
  __shared__ __align__(16) float Bs[2][BK * LDB];

  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * p.k_chunk;
  const int kend = min(p.K, kbeg + p.k_chunk);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  float4 ra[BM / 64], rb[BN / 64];
  load_tile<A_KC, BM>(p.A, p.a_rows, p.a_vec, m0, p.M, kbeg, kend, ra);
  load_tile<B_KC, BN>(p.B, p.b_rows, p.b_vec, n0, p.N, kbeg, kend, rb);
  store_tile<A_KC, BM>(As[0], ra);
  store_tile<B_KC, BN>(Bs[0], rb);
  __syncthreads();

  int buf = 0;
  for (int k0 = kbeg; k0 < kend; k0 += BK) {
    const bool has_next = (k0 + BK) < kend;
    if (has_next) {
      load_tile<A_KC, BM>(p.A, p.a_rows, p.a_vec, m0, p.M, k0 + BK, kend, ra);
      load_tile<B_KC, BN>(p.B, p.b_rows, p.b_vec, n0, p.N, k0 + BK, kend, rb);
    }
    const float* as = As[buf];
    const float* bs = Bs[buf];
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[TM], b[TN];
#pragma unroll
      for (int h = 0; h < TM / 4; ++h) {
        float4 v = *reinterpret_cast<const float4*>(&as[kk * LDA + h * 64 + ty * 4]);
        a[h * 4 + 0] = v.x; a[h * 4 + 1] = v.y; a[h * 4 + 2] = v.z; a[h * 4 + 3] = v.w;
      }
#pragma unroll
      for (int h = 0; h < TN / 4; ++h) {
        float4 v = *reinterpret_cast<const float4*>(&bs[kk * LDB + h * 64 + tx * 4]);
        b[h * 4 + 0] = v.x; b[h * 4 + 1] = v.y; b[h * 4 + 2] = v.z; b[h * 4 + 3] = v.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (has_next) {
      store_tile<A_KC, BM>(As[buf ^ 1], ra);
      store_tile<B_KC, BN>(Bs[buf ^ 1], rb);
    }
    __syncthreads();
    buf ^= 1;
  }

  // epilogue
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int m = m0 + (i >> 2) * 64 + ty * 4 + (i & 3);
    if (m >= p.M) continue;
#pragma unroll
    for (int h = 0; h < TN / 4; ++h) {
      const int n = n0 + h * 64 + tx * 4;
      if (n >= p.N) continue;
      float v[4] = {acc[i][h * 4 + 0], acc[i][h * 4 + 1], acc[i][h * 4 + 2], acc[i][h * 4 + 3]};
      if (p.splitk > 1) {
        float* dst = p.partial + ((size_t)blockIdx.z * p.M + m) * p.N + n;
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (n + e < p.N) dst[e] = v[e];
      } else {
        float* dst = p.C + p.c_rows.off(m) + n;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (n + e < p.N) {
            float o = v[e];
            if (p.bias1) o += __ldg(p.bias1 + n + e);
            if (p.bias2 && (n + e) < p.bias2_n) o += __ldg(p.bias2 + n + e);
            if (p.accumulate) o += dst[e];
            dst[e] = o;
          }
        }
      }
    }
  }
}

// C(m,n) (+)= sum_z partial[z][m][n] + bias  — fixed summation order => deterministic wgrad.
__global__ void splitk_reduce_kernel(const float* __restrict__ partial, int splitk, int M, int N, float* C,
                                     RowMap c_rows, const float* bias1, const float* bias2, int bias2_n,
                                     int accumulate) {
  const size_t total = (size_t)M * N;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    int m = (int)(idx / N), n = (int)(idx - (size_t)m * N);
    float s = 0.f;
    for (int z = 0; z < splitk; ++z) s += partial[(size_t)z * total + idx];
    if (bias1) s += bias1[n];
    if (bias2 && n < bias2_n) s += bias2[n];
    float* dst = C + c_rows.off(m) + n;
    if (accumulate) s += *dst;
    *dst = s;
  }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
inline bool rows_vec_ok(const float* base, const RowMap& r) {
  return aligned16(base) && (r.s_outer % 4 == 0) && (r.s_inner % 4 == 0);
}

struct Plan {
  int tile;  // 128 or 64
  int splitk;
  int k_chunk;
};

Plan make_plan(int M, int N, int K, size_t scratch_bytes, bool have_scratch) {
  Plan pl;
  const long t128 = (long)((M + 127) / 128) * ((N + 127) / 128);
  const long t64 = (long)((M + 63) / 64) * ((N + 63) / 64);
  pl.tile = (t128 >= 120) ? 128 : 64;
  pl.splitk = 1;
  const long tiles = pl.tile == 128 ? t128 : t64;
  if (have_scratch && tiles < 120 && K >= 1024) {
    int want = (int)((296 + tiles - 1) / tiles);
    int maxk = K / 256;  // keep >= 256 of K per split
    int s = want < maxk ? want : maxk;
    size_t per = (size_t)M * N * sizeof(float);
    while (s > 1 && per * s > scratch_bytes) --s;
    if (s > 1) pl.splitk = s;
  }
  int chunk = (K + pl.splitk - 1) / pl.splitk;
  chunk = ((chunk + BK - 1) / BK) * BK;
  pl.k_chunk = chunk;
  pl.splitk = (K + chunk - 1) / chunk;
  if (pl.splitk < 1) pl.splitk = 1;
  return pl;
}

template <int BM, int BN>
void launch_tile(const GemmDev& d, bool a_kc, bool b_kc, dim3 grid, cudaStream_t s) {
  if (a_kc && b_kc)
    gemm_f32_kernel<true, true, BM, BN><<<grid, NTHREADS, 0, s>>>(d);
  else if (a_kc && !b_kc)
    gemm_f32_kernel<true, false, BM, BN><<<grid, NTHREADS, 0, s>>>(d);
  else if (!a_kc && b_kc)
    gemm_f32_kernel<false, true, BM, BN><<<grid, NTHREADS, 0, s>>>(d);
  else
    gemm_f32_kernel<false, false, BM, BN><<<grid, NTHREADS, 0, s>>>(d);
}

}  // namespace

void gemm_splitk_plan(int M, int N, int K, void* scratch, size_t scratch_bytes, int* splitk, int* k_chunk) {
  const Plan pl = make_plan(M, N, K > 0 ? K : 1, scratch_bytes, scratch != nullptr);
  *splitk = K > 0 ? pl.splitk : 1;
  *k_chunk = K > 0 ? pl.k_chunk : BK;
}

int launch_splitk_reduce(const float* partial, int splitk, int M, int N, float* C, const RowMap& c_rows,
                         const float* bias1, const float* bias2, int bias2_n, int accumulate, cudaStream_t stream) {
  size_t total = (size_t)M * N;
  int blocks = (int)((total + 255) / 256);
  if (blocks > NUM_SMS * 8) blocks = NUM_SMS * 8;
  if (blocks < 1) blocks = 1;
  splitk_reduce_kernel<<<blocks, 256, 0, stream>>>(partial, splitk, M, N, C, c_rows, bias1, bias2, bias2_n, accumulate);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

size_t gemm_scratch_bytes(int M, int N, int K) {
  // worst case the planner may want: up to 296 tiles' worth of splits, bounded by K/256
  const long t64 = (long)((M + 63) / 64) * ((N + 63) / 64);
  if (t64 >= 120 || K < 1024) return 0;
  int want = (int)((296 + t64 - 1) / t64);
  int maxk = K / 256;
  int s = want < maxk ? want : maxk;
  if (s <= 1) return 0;
  return (size_t)s * M * N * sizeof(float);
}

int launch_gemm(const GemmParams& p, void* scratch, size_t scratch_bytes, cudaStream_t stream) {
  if (p.M <= 0 || p.N <= 0) return B200RNN_OK;
  if (!p.A || !p.B || !p.C) {
    set_error("gemm: null operand");
    return B200RNN_ERR_INVALID;
  }
  if (p.tc_ws && gemm_tc_eligible(p, p.tc_ws_bytes)) return launch_gemm_tc(p, p.tc_ws, p.tc_ws_bytes, stream);
  if (p.tc_ready) {
    set_error("gemm: a streamed launch needs the tensor-core path");
    return B200RNN_ERR_INVALID;
  }
  GemmDev d;
  d.A = p.A; d.a_rows = p.a_rows;
  d.B = p.B; d.b_rows = p.b_rows;
  d.C = p.C; d.c_rows = p.c_rows;
  d.M = p.M; d.N = p.N; d.K = p.K;
  d.bias1 = p.bias1; d.bias2 = p.bias2; d.bias2_n = p.bias2_n;
  d.accumulate = p.accumulate;
  d.a_vec = rows_vec_ok(p.A, p.a_rows);
  d.b_vec = rows_vec_ok(p.B, p.b_rows);
  static const bool debug = getenv("B200RNN_DEBUG") != nullptr;
  // the forward input projection on this GEMM: A read through its row map ("rows"), or a dense copy of it. Its own
  // line: "forward x-projection" names the tensor-core projections
  if (debug && p.a_route)
    fprintf(stderr, "[b200rnn] ffma x-projection: M=%d N=%d K=%d a=%s loads=%s\n", p.M, p.N, p.K,
            strcmp(p.a_route, "tma") ? p.a_route : "rows", d.a_vec ? "vec4" : "scalar");
  Plan pl = make_plan(p.M, p.N, p.K > 0 ? p.K : 1, scratch_bytes, scratch != nullptr);
  d.splitk = pl.splitk;
  d.k_chunk = pl.k_chunk;
  d.partial = static_cast<float*>(scratch);
  if (p.K <= 0) {  // empty contraction: C = bias (+C)
    d.splitk = 1;
    d.k_chunk = BK;
  }
  ProfScope prof(PROF_GEMM, stream);
  dim3 grid((p.N + pl.tile - 1) / pl.tile, (p.M + pl.tile - 1) / pl.tile, d.splitk);
  if (pl.tile == 128)
    launch_tile<128, 128>(d, p.a_kcontig, p.b_kcontig, grid, stream);
  else
    launch_tile<64, 64>(d, p.a_kcontig, p.b_kcontig, grid, stream);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  if (d.splitk > 1) {
    size_t total = (size_t)p.M * p.N;
    int blocks = (int)((total + 255) / 256);
    if (blocks > NUM_SMS * 8) blocks = NUM_SMS * 8;
    splitk_reduce_kernel<<<blocks, 256, 0, stream>>>(d.partial, d.splitk, p.M, p.N, p.C, p.c_rows, p.bias1,
                                                     p.bias2, p.bias2_n, p.accumulate);
    B200_CUDA_CHECK(cudaGetLastError());
    count_launch();
  }
  return B200RNN_OK;
}

}  // namespace b200rnn
