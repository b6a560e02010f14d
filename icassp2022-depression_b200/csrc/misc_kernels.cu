// misc_kernels.cu — dropout (K7), weight transpose, bias-gradient reduction. All HBM-bound, coalesced,
// grid sized in multiples of the SM count.
#include "misc_kernels.cuh"

namespace b200rnn {

namespace {


// Inter-layer dropout, nn.GRU/nn.LSTM semantics (rnn.py:857-860, :1233-1236): Bernoulli(1-p) keep mask,
// kept values scaled by 1/(1-p). One Philox call yields the mask of 4 consecutive elements.
__global__ void rng_setup_kernel(uint64_t* hdr, uint64_t seed, uint64_t offset, uint64_t* state_dev,
                                 uint64_t consume) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    if (state_dev) {
      seed = state_dev[0];
      offset = state_dev[1];
      state_dev[1] = offset + consume;
    }
    hdr[0] = seed;
    hdr[1] = offset;
  }
}

__global__ void dropout_kernel(const float* __restrict__ in, float* __restrict__ out, size_t n, float p,
                               float scale, const uint64_t* __restrict__ hdr, uint32_t stream_id) {
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

__global__ void dropout_split_kernel(const float* __restrict__ in, float* __restrict__ out, float* __restrict__ hi,
                                     float* __restrict__ lo, size_t n, float p, float scale,
                                     const uint64_t* __restrict__ hdr, uint32_t stream_id) {
  const uint64_t seed = hdr[0], offset = hdr[1];
  const size_t nquad = n / 4;
  const uint32_t thr = (uint32_t)fminf(p * 4294967296.0f, 4294967295.0f);
  for (size_t qd = blockIdx.x * (size_t)blockDim.x + threadIdx.x; qd < nquad;
       qd += (size_t)gridDim.x * blockDim.x) {
    Philox4 r = philox4x32_10(seed, offset + qd, (uint64_t)stream_id);  // same stream as dropout_kernel
    float4 v = *reinterpret_cast<const float4*>(in + qd * 4);
    v.x = r.x >= thr ? v.x * scale : 0.f;
    v.y = r.y >= thr ? v.y * scale : 0.f;
    v.z = r.z >= thr ? v.z * scale : 0.f;
    v.w = r.w >= thr ? v.w * scale : 0.f;
    if (out) *reinterpret_cast<float4*>(out + qd * 4) = v;
    float4 h, l;
    uint32_t t;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(v.x)); h.x = __uint_as_float(t); l.x = v.x - h.x;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(v.y)); h.y = __uint_as_float(t); l.y = v.y - h.y;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(v.z)); h.z = __uint_as_float(t); l.z = v.z - h.z;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(t) : "f"(v.w)); h.w = __uint_as_float(t); l.w = v.w - h.w;
    *reinterpret_cast<float4*>(hi + qd * 4) = h;
    *reinterpret_cast<float4*>(lo + qd * 4) = l;
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

}  // namespace

int launch_rng_setup(uint64_t* hdr, uint64_t seed, uint64_t offset, uint64_t* state_dev, uint64_t consume,
                     cudaStream_t stream) {
  rng_setup_kernel<<<1, 32, 0, stream>>>(hdr, seed, offset, state_dev, consume);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

int launch_dropout(const float* in, float* out, size_t n, float p, const uint64_t* hdr, uint32_t stream_id,
                   cudaStream_t stream) {
  if (n == 0) return B200RNN_OK;
  const float scale = p < 1.f ? 1.f / (1.f - p) : 0.f;
  size_t nquad = (n + 3) / 4;
  int blocks = (int)((nquad + 255) / 256);
  if (blocks > NUM_SMS * 8) blocks = NUM_SMS * 8;
  dropout_kernel<<<blocks, 256, 0, stream>>>(in, out, n, p, scale, hdr, stream_id);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

int launch_dropout_split(const float* in, float* out, float* hi, float* lo, size_t n, float p, const uint64_t* hdr,
                         uint32_t stream_id, cudaStream_t stream) {
  if (n == 0) return B200RNN_OK;
  if (n % 4 != 0) {
    set_error("dropout_split: element count must be a multiple of 4");
    return B200RNN_ERR_INVALID;
  }
  const float scale = p < 1.f ? 1.f / (1.f - p) : 0.f;
  size_t nquad = n / 4;
  int blocks = (int)((nquad + 255) / 256);
  if (blocks > NUM_SMS * 8) blocks = NUM_SMS * 8;
  dropout_split_kernel<<<blocks, 256, 0, stream>>>(in, out, hi, lo, n, p, scale, hdr, stream_id);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}


int launch_bias_reduce(const float* part, int nslices, int mode, int H, float* db_ih, float* db_hh,
                       int accumulate, cudaStream_t stream) {
  const int G = mode == B200RNN_GRU ? 3 : 4;
  const int GH = G * H;
  bias_reduce_kernel<<<(GH + 127) / 128, 128, 0, stream>>>(part, nslices, mode, H, db_ih, db_hh, accumulate);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

}  // namespace b200rnn
