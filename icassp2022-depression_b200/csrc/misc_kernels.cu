// misc_kernels.cu — dropout (K7), weight transpose, bias-gradient reduction. All HBM-bound, coalesced,
// grid sized in multiples of the SM count. Plus the one-CTA batch-slot order of a ragged batch.
#include "misc_kernels.cuh"

namespace b200rnn {

namespace {


// Inter-layer dropout, nn.GRU/nn.LSTM semantics (rnn.py:857-860, :1233-1236): Bernoulli(1-p) keep mask,
// kept values scaled by 1/(1-p). One Philox call yields the mask of 4 consecutive elements.
__global__ void rng_setup_kernel(uint64_t* hdr, uint64_t seed, uint64_t offset, uint64_t* state_dev,
                                 uint64_t consume, uint64_t skip) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    if (state_dev) {
      seed = state_dev[0];
      offset = state_dev[1];
      state_dev[1] = offset + consume;
    }
    hdr[0] = seed;
    hdr[1] = offset + skip;
  }
}

__global__ void dropout_kernel(const float* __restrict__ in, float* __restrict__ out, size_t n, float p,
                               float scale, const uint64_t* __restrict__ hdr, uint32_t stream_id,
                               int* __restrict__ clear, int nclear) {
  if (blockIdx.x == 0)
    for (int i = threadIdx.x; i < nclear; i += blockDim.x) clear[i] = 0;
  const uint64_t seed = hdr[0], offset = hdr[1];
  const size_t nquad = (n + 3) / 4;
  // keep iff u >= p where u = x * 2^-32 in [0,1)
  const uint32_t thr = (uint32_t)fminf(p * 4294967296.0f, 4294967295.0f);
  for (size_t qd = blockIdx.x * (size_t)blockDim.x + threadIdx.x; qd < nquad;
       qd += (size_t)gridDim.x * blockDim.x) {
    Philox4 r = philox4x32_10(seed, offset + qd, (uint64_t)stream_id);
    const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
    const size_t i0 = qd * 4;
    if (i0 + 3 < n && ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15u) == 0) {
      float4 v = *reinterpret_cast<const float4*>(in + i0);
      v.x = rr[0] >= thr ? v.x * scale : 0.f;
      v.y = rr[1] >= thr ? v.y * scale : 0.f;
      v.z = rr[2] >= thr ? v.z * scale : 0.f;
      v.w = rr[3] >= thr ? v.w * scale : 0.f;
      *reinterpret_cast<float4*>(out + i0) = v;
    } else {
      for (int e = 0; e < 4 && i0 + e < n; ++e) out[i0 + e] = rr[e] >= thr ? in[i0 + e] * scale : 0.f;
    }
  }
}

// Rank of row i = #{j : len_j > len_i} + #{j < i : len_j == len_i}: a permutation, deterministic, no atomics. The
// lengths go through shared memory in tiles of ORDER_TILE; B^2 compares in all (16K at B = 128).
constexpr int ORDER_TILE = 1024;

__global__ void length_order_kernel(const int* __restrict__ lengths, int B, int* __restrict__ order) {
  __shared__ int tile[ORDER_TILE];
  for (int i0 = 0; i0 < B; i0 += blockDim.x) {  // every thread runs every iteration (the barriers below)
    const int i = i0 + threadIdx.x;
    const int li = i < B ? lengths[i] : 0;
    int rank = 0;
    for (int j0 = 0; j0 < B; j0 += ORDER_TILE) {
      const int n = min(ORDER_TILE, B - j0);
      __syncthreads();
      for (int k = threadIdx.x; k < n; k += blockDim.x) tile[k] = lengths[j0 + k];
      __syncthreads();
      for (int k = 0; k < n; ++k) {
        const int lj = tile[k];
        rank += (lj > li || (lj == li && j0 + k < i)) ? 1 : 0;
      }
    }
    if (i < B) order[rank] = i;
  }
}

__global__ void initial_state_rows_kernel(const float* __restrict__ dgates, const float* __restrict__ dghn, int mode,
                                          int B, int T, int H, int reverse, const int* __restrict__ lengths,
                                          float* __restrict__ out) {
  const int GH = (mode == B200RNN_GRU ? 3 : 4) * H;
  const size_t n = (size_t)B * GH;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / GH), c = (int)(i % GH);
    const int t = reverse ? (lengths ? min(max(lengths[b], 0), T) : T) - 1 : 0;
    float v = 0.f;
    if (t >= 0) {
      const size_t row = (size_t)t * B + b;
      v = (mode == B200RNN_GRU && c >= 2 * H) ? dghn[row * H + (c - 2 * H)] : dgates[row * GH + c];
    }
    out[i] = v;
  }
}

__global__ void valid_rows_kernel(const float* __restrict__ src, RowMap rows, int T, int B, int C,
                                  const int* __restrict__ lengths, float* __restrict__ dst) {
  const size_t n = (size_t)T * B * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / C), c = (int)(i % C);
    const int t = r / B, b = r - t * B;
    dst[i] = t < lengths[b] ? src[rows.off(r) + c] : 0.f;
  }
}

__global__ void bias_reduce_kernel(const float* __restrict__ part, int nslices, int mode, int H, float* db_ih,
                                   float* db_hh, int accumulate) {
  const int G = mode == B200RNN_GRU ? 3 : 4;
  const int GH = G * H, W = (G + 1) * H;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= GH) return;
  float s = 0.f, sn = 0.f;
  const bool gru_n = (mode == B200RNN_GRU) && c >= 2 * H;
  int k = 0;
  for (; k + 8 <= nslices; k += 8) {  // 8 independent loads in flight, added in a fixed order => deterministic
    float v[8], vn[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      v[u] = part[(size_t)(k + u) * W + c];
      vn[u] = gru_n ? part[(size_t)(k + u) * W + GH + (c - 2 * H)] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      s += v[u];
      sn += vn[u];
    }
  }
  for (; k < nslices; ++k) {
    s += part[(size_t)k * W + c];
    if (gru_n) sn += part[(size_t)k * W + GH + (c - 2 * H)];
  }
  const float hh = gru_n ? sn : s;
  if (db_ih) db_ih[c] = accumulate ? db_ih[c] + s : s;
  if (db_hh) db_hh[c] = accumulate ? db_hh[c] + hh : hh;
}

// Elman: db_ih = db_hh = the column sums of the per-slice partials [nslices][H] of dpre, in the same fixed order
__global__ void elman_bias_reduce_kernel(const float* __restrict__ part, int nslices, int H, float* db_ih,
                                         float* db_hh, int accumulate) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  float s = 0.f;
  int k = 0;
  for (; k + 8 <= nslices; k += 8) {
    float v[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) v[u] = part[(size_t)(k + u) * H + c];
#pragma unroll
    for (int u = 0; u < 8; ++u) s += v[u];
  }
  for (; k < nslices; ++k) s += part[(size_t)k * H + c];
  if (db_ih) db_ih[c] = accumulate ? db_ih[c] + s : s;
  if (db_hh) db_hh[c] = accumulate ? db_hh[c] + s : s;
}

}  // namespace

int launch_rng_setup(uint64_t* hdr, uint64_t seed, uint64_t offset, uint64_t* state_dev, uint64_t consume,
                     cudaStream_t stream, uint64_t skip) {
  rng_setup_kernel<<<1, 32, 0, stream>>>(hdr, seed, offset, state_dev, consume, skip);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

int launch_dropout(const float* in, float* out, size_t n, float p, const uint64_t* hdr, uint32_t stream_id,
                   cudaStream_t stream, int* clear, int nclear) {
  if (n == 0) return B200RNN_OK;
  const float scale = p < 1.f ? 1.f / (1.f - p) : 0.f;
  size_t nquad = (n + 3) / 4;
  int blocks = (int)((nquad + 255) / 256);
  if (blocks > NUM_SMS * 8) blocks = NUM_SMS * 8;
  dropout_kernel<<<blocks, 256, 0, stream>>>(in, out, n, p, scale, hdr, stream_id, clear, clear ? nclear : 0);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

int launch_length_order(const int* lengths, int B, int* order, cudaStream_t stream) {
  if (B <= 0) return B200RNN_OK;
  const int threads = B < ORDER_TILE ? (B + 31) / 32 * 32 : ORDER_TILE;
  length_order_kernel<<<1, threads, 0, stream>>>(lengths, B, order);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

int launch_initial_state_rows(const float* dgates, const float* dghn, int mode, int B, int T, int H, bool reverse,
                              const int* lengths, float* out, cudaStream_t stream) {
  if (is_elman(mode)) {  // G*H = H columns and no GRU n block: the LSTM rows of the kernel, H / 4 units per gate
    if (H % 4) {
      set_error("initial_state_rows: Elman hidden_size %d is not a multiple of 4", H);
      return B200RNN_ERR_INVALID;
    }
    mode = B200RNN_LSTM;
    H /= 4;
  }
  const size_t n = (size_t)B * (mode == B200RNN_GRU ? 3 : 4) * H;
  if (n == 0) return B200RNN_OK;
  int blocks = (int)((n + 255) / 256);
  if (blocks > NUM_SMS * 4) blocks = NUM_SMS * 4;
  initial_state_rows_kernel<<<blocks, 256, 0, stream>>>(dgates, dghn, mode, B, T, H, reverse ? 1 : 0, lengths, out);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

int launch_valid_rows(const float* src, const RowMap& rows, int T, int B, int C, const int* lengths, float* dst,
                      cudaStream_t stream) {
  const size_t n = (size_t)T * B * C;
  if (n == 0) return B200RNN_OK;
  int blocks = (int)((n + 255) / 256);
  if (blocks > NUM_SMS * 8) blocks = NUM_SMS * 8;
  valid_rows_kernel<<<blocks, 256, 0, stream>>>(src, rows, T, B, C, lengths, dst);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

int launch_bias_reduce(const float* part, int nslices, int mode, int H, float* db_ih, float* db_hh,
                       int accumulate, cudaStream_t stream) {
  if (is_elman(mode)) {
    elman_bias_reduce_kernel<<<(H + 127) / 128, 128, 0, stream>>>(part, nslices, H, db_ih, db_hh, accumulate);
    B200_CUDA_CHECK(cudaGetLastError());
    count_launch();
    return B200RNN_OK;
  }
  const int G = mode == B200RNN_GRU ? 3 : 4;
  const int GH = G * H;
  bias_reduce_kernel<<<(GH + 127) / 128, 128, 0, stream>>>(part, nslices, mode, H, db_ih, db_hh, accumulate);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

}  // namespace b200rnn
