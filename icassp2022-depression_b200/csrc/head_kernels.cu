// head_kernels.cu — the small dense shells on either side of the encoders inside the fuse step, fused into a
// handful of kernels (SURVEY.md 8f rank 1 "attention pooling as one small kernel", rank 3 "fused optimiser + loss").
// They replace ~45 tiny framework launches per step of fuse_net_whole.py:336-366, 445-456:
//   attention_pool_kernel : attention_net_with_w (text_bilstm_whole.py:74-99 / fuse_net_whole.py:310-334)
//   mlp_dropout_kernel    : Dropout -> Linear -> ReLU -> Dropout   (fc_out / fc_audio of fusion_net, :270-275, :288-293)
//   fuse_loss_grad_kernel : Softmax(fc_final(concat)), MyLoss two-head CE, and d loss / d fc_final.0.weight (:368-395)
//   adam_kernel           : torch.optim.Adam step (no weight decay / amsgrad) over a flat parameter range (:416, :456)
// All are latency-bound dwarfs (a few KB..MB); the point is launch count, not bandwidth.
#include "common.cuh"
#include "misc_kernels.cuh"

namespace b200rnn {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// out[i] = W[i,:] . x (+ bias) for the rows this warp owns (i = warp, warp + nw, ...), FOUR rows per pass so that a lane
// keeps 4 x (H/32) independent L2 loads in flight instead of one dependent round trip per row (the first version spent
// ~13 us of a 34 us launch in this loop at H = 256)
template <bool RELU>
__device__ __forceinline__ void warp_matvec_rows(const float* __restrict__ W, const float* __restrict__ bias,
                                                 const float* x_s, float* out_s, int H, int warp, int nw, int lane) {
  for (int i = warp; i < H; i += 4 * nw) {
    float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 2
    for (int j = lane; j < H; j += 32) {
      const float xv = x_s[j];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int ii = i + r * nw;
        if (ii < H) s[r] += __ldg(W + (size_t)ii * H + j) * xv;
      }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int ii = i + r * nw;
      const float v = warp_sum(s[r]);
      if (lane == 0 && ii < H) {
        const float o = v + bias[ii];
        out_s[ii] = RELU ? fmaxf(o, 0.f) : o;
      }
    }
  }
}

// keep-mask of element `idx` of dropout stream `stream_id` (same Philox layout as dropout_kernel: 4 per call)
__device__ __forceinline__ float keep_scale(const uint64_t* hdr, uint32_t stream_id, size_t idx, uint32_t thr,
                                            float scale) {
  Philox4 r = philox4x32_10(hdr[0], hdr[1] + (idx >> 2), (uint64_t)stream_id);
  const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
  return rr[idx & 3] >= thr ? scale : 0.f;
}

// ---- attention pooling: one CTA per batch row ------------------------------------------------------------
//   seq   : [T,B,2H] addressed t*s_t + b*s_b + c   (fwd | rev halves)
//   h_n   : [NS,B,H]  final hidden states (all layers / directions), summed
//   ctx[b] = sum_t softmax_t( ReLU(W_a hsum + b_a) . tanh(h_t) ) * h_t,   h_t = seq[t,b,:H] + seq[t,b,H:]
__global__ void attention_pool_kernel(const float* __restrict__ seq, long long s_t, long long s_b,
                                      const float* __restrict__ h_n, int NS, int B, int T, int H,
                                      const float* __restrict__ w_a, const float* __restrict__ b_a,
                                      float* __restrict__ ctx) {
  extern __shared__ float sm[];
  float* hsum = sm;          // [H]
  float* q = sm + H;         // [H]
  float* score = sm + 2 * H; // [T]
  __shared__ float red[2];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;

  for (int j = tid; j < H; j += blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < NS; ++k) s += h_n[((size_t)k * B + b) * H + j];
    hsum[j] = s;
  }
  __syncthreads();
  warp_matvec_rows<true>(w_a, b_a, hsum, q, H, warp, nw, lane);  // q = ReLU(W_a hsum + b_a)
  __syncthreads();
  const float* row0 = seq + (long long)b * s_b;
  for (int t = warp; t < T; t += nw) {  // scores, one warp per time step
    const float* r = row0 + (long long)t * s_t;
    float s = 0.f;
#pragma unroll 8
    for (int j = lane; j < H; j += 32) s += q[j] * tanhf(__ldg(r + j) + __ldg(r + H + j));
    s = warp_sum(s);
    if (lane == 0) score[t] = s;
  }
  __syncthreads();
  if (warp == 0) {  // softmax over T
    float m = -INFINITY;
    for (int t = lane; t < T; t += 32) m = fmaxf(m, score[t]);
    m = warp_max(m);
    float z = 0.f;
    for (int t = lane; t < T; t += 32) {
      const float e = expf(score[t] - m);
      score[t] = e;
      z += e;
    }
    z = warp_sum(z);
    if (lane == 0) red[0] = 1.f / z;
  }
  __syncthreads();
  const float inv = red[0];
  for (int j = tid; j < H; j += blockDim.x) {
    float a = 0.f;
#pragma unroll 8
    for (int t = 0; t < T; ++t) {
      const float* r = row0 + (long long)t * s_t;
      a += score[t] * (__ldg(r + j) + __ldg(r + H + j));
    }
    ctx[(size_t)b * H + j] = a * inv;
  }
}

// ---- backward of the attention pooling (text_bilstm_whole.py:74-99 under loss.backward()): one CTA per batch row ------
//   forward (recomputed): hsum = sum_k h_n[k,b]; qpre = W hsum + b; q = ReLU(qpre); h_t = seq[t,b,:H] + seq[t,b,H:];
//                         s_t = q . tanh(h_t); a = softmax_t(s); ctx = sum_t a_t h_t
//   backward: da_t = dctx . h_t; ds_t = a_t (da_t - sum_u a_u da_u); dq = sum_t ds_t tanh(h_t);
//             dh_t = a_t dctx + ds_t q (1 - tanh(h_t)^2)  -> both halves of dseq[t,b,:]
//             dqpre = dq [qpre > 0]; dhsum = W^T dqpre -> every dh_n[k,b,:];  dW = sum_b dqpre hsum^T, db = sum_b dqpre
//   (the two batch reductions are left to the caller: dqpre / hsum rows go to [B,H] buffers, dW is one small GEMM)
__global__ void __launch_bounds__(256)
    attention_pool_bwd_kernel(const float* __restrict__ seq, long long s_t, long long s_b, const float* __restrict__ h_n,
                              int NS, int B, int T, int H, const float* __restrict__ w_a, const float* __restrict__ b_a,
                              const float* __restrict__ dctx, float* __restrict__ dseq, long long d_t, long long d_b,
                              float* __restrict__ dh_n, float* __restrict__ dqpre_out, float* __restrict__ hsum_out) {
  extern __shared__ float sm[];
  float* hsum = sm;            // [H]
  float* qpre = hsum + H;      // [H]
  float* dc = qpre + H;        // [H] dctx row
  float* dqp = dc + H;         // [H]
  float* score = dqp + H;      // [T] -> a_t
  float* ds = score + T;       // [T]
  float* hs = ds + T;          // [T][H] h_t
  __shared__ float red[2];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const float* row0 = seq + (long long)b * s_b;
  for (int j = tid; j < H; j += blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < NS; ++k) s += h_n[((size_t)k * B + b) * H + j];
    hsum[j] = s;
    dc[j] = dctx[(size_t)b * H + j];
    if (hsum_out) hsum_out[(size_t)b * H + j] = s;
  }
#pragma unroll 8
  for (int idx = tid; idx < T * H; idx += blockDim.x) {
    const int t = idx / H, j = idx - t * H;
    const float* r = row0 + (long long)t * s_t;
    hs[idx] = __ldg(r + j) + __ldg(r + H + j);
  }
  __syncthreads();
  warp_matvec_rows<false>(w_a, b_a, hsum, qpre, H, warp, nw, lane);  // qpre = W hsum + b
  __syncthreads();
  for (int t = warp; t < T; t += nw) {  // scores and da_t, one warp per time step
    float s = 0.f, da = 0.f;
    for (int j = lane; j < H; j += 32) {
      const float h = hs[t * H + j];
      s += fmaxf(qpre[j], 0.f) * tanhf(h);
      da += dc[j] * h;
    }
    s = warp_sum(s);
    da = warp_sum(da);
    if (lane == 0) {
      score[t] = s;
      ds[t] = da;
    }
  }
  __syncthreads();
  if (warp == 0) {  // softmax over T, then ds_t = a_t (da_t - sum_u a_u da_u)
    float m = -INFINITY;
    for (int t = lane; t < T; t += 32) m = fmaxf(m, score[t]);
    m = warp_max(m);
    float z = 0.f;
    for (int t = lane; t < T; t += 32) {
      const float e = expf(score[t] - m);
      score[t] = e;
      z += e;
    }
    z = warp_sum(z);
    const float inv = 1.f / z;
    float dot = 0.f;
    for (int t = lane; t < T; t += 32) {
      const float a = score[t] * inv;
      score[t] = a;
      dot += a * ds[t];
    }
    dot = warp_sum(dot);
    for (int t = lane; t < T; t += 32) ds[t] = score[t] * (ds[t] - dot);
  }
  __syncthreads();
  for (int j = tid; j < H; j += blockDim.x) {
    const float q = fmaxf(qpre[j], 0.f), dcj = dc[j];
    float dq = 0.f;
    for (int t = 0; t < T; ++t) {
      const float th = tanhf(hs[t * H + j]);
      dq += ds[t] * th;
      const float dh = score[t] * dcj + ds[t] * q * (1.f - th * th);
      float* o = dseq + (long long)t * d_t + (long long)b * d_b;
      o[j] = dh;
      o[H + j] = dh;
    }
    const float v = qpre[j] > 0.f ? dq : 0.f;
    dqp[j] = v;
    if (dqpre_out) dqpre_out[(size_t)b * H + j] = v;
  }
  __syncthreads();
  for (int i = tid; i < H; i += blockDim.x) {  // dhsum = W^T dqpre (coalesced over i), 16 independent loads in flight
    float s0 = 0.f, s1 = 0.f;
    int j = 0;
    for (; j + 16 <= H; j += 16) {
      float wv[16];
#pragma unroll
      for (int u = 0; u < 16; ++u) wv[u] = __ldg(w_a + (size_t)(j + u) * H + i);
#pragma unroll
      for (int u = 0; u < 16; u += 2) {
        s0 += wv[u] * dqp[j + u];
        s1 += wv[u + 1] * dqp[j + u + 1];
      }
    }
    for (; j < H; ++j) s0 += __ldg(w_a + (size_t)j * H + i) * dqp[j];
    const float s = s0 + s1;
    for (int k = 0; k < NS; ++k) dh_n[((size_t)k * B + b) * H + i] = s;
  }
  (void)red;
}

// ---- out = D2(ReLU(W D1(x) + bias)) as a small tiled GEMM: CTA tile = 32 outputs x 32 batch rows ---------------
// Both operand tiles are staged in shared memory with bulk coalesced loads (no dependent global-load chains; the
// first version, one warp-dot per output, spent its time waiting on one L2 round trip per 32 columns).
constexpr int MLP_TI = 32, MLP_TB = 32;
__global__ void __launch_bounds__(256)
    mlp_dropout_kernel(const float* __restrict__ x, int B, int n, const float* __restrict__ W,
                       const float* __restrict__ bias, float* __restrict__ out, int training, float p,
                       const uint64_t* __restrict__ hdr, uint32_t stream_id) {
  extern __shared__ float sm[];
  const int ld = n + 1;                // +1: conflict-free column walks
  float* Ws = sm;                      // [MLP_TI][ld]
  float* xs = sm + MLP_TI * ld;        // [MLP_TB][ld]
  const int i0 = blockIdx.x * MLP_TI, b0 = blockIdx.y * MLP_TB, tid = threadIdx.x;
  const bool drop = training && p > 0.f;
  const uint32_t thr = (uint32_t)fminf(p * 4294967296.0f, 4294967295.0f);
  const float scale = p < 1.f ? 1.f / (1.f - p) : 0.f;
  for (int idx = tid; idx < MLP_TI * n; idx += blockDim.x) {
    const int r = idx / n, j = idx - r * n;
    Ws[r * ld + j] = (i0 + r < n) ? __ldg(W + (size_t)(i0 + r) * n + j) : 0.f;
  }
  for (int idx = tid; idx < MLP_TB * n; idx += blockDim.x) {
    const int r = idx / n, j = idx - r * n, b = b0 + r;
    float v = 0.f;
    if (b < B) {
      v = x[(size_t)b * n + j];
      if (drop) v *= keep_scale(hdr, stream_id, (size_t)b * n + j, thr, scale);
    }
    xs[r * ld + j] = v;
  }
  __syncthreads();
  const int ti = tid & 31, tb = tid >> 5;  // output column ti, batch rows tb, tb+8, tb+16, tb+24
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const float* wrow = Ws + ti * ld;
  for (int j = 0; j < n; ++j) {
    const float w = wrow[j];
#pragma unroll
    for (int r = 0; r < 4; ++r) acc[r] = fmaf(w, xs[(tb + 8 * r) * ld + j], acc[r]);
  }
  const int i = i0 + ti;
  if (i < n) {
    const float bi = bias[i];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int b = b0 + tb + 8 * r;
      if (b < B) {
        float v = fmaxf(acc[r] + bi, 0.f);
        if (drop) v *= keep_scale(hdr, stream_id + 1, (size_t)b * n + i, thr, scale);
        out[(size_t)b * n + i] = v;
      }
    }
  }
}

// ---- two-head cross entropy on the halves of fc_final.0.weight, its gradient, and the fused softmax output ------
//   W [2, Ht+Ha];  loss = CE(tf W[:, :Ht]^T, y) + CE(af W[:, Ht:]^T, y)  (mean over B)
//   dW (+)= d loss / dW ;  probs = softmax(cat(tf,af) W^T)
constexpr int LOSS_THREADS = 512;
constexpr int LOSS_MAXF = 512;   // Ht + Ha
constexpr int LOSS_CPL = LOSS_MAXF / 32;  // feature columns per lane
__global__ void __launch_bounds__(LOSS_THREADS)
    fuse_loss_grad_kernel(const float* __restrict__ tf, int Ht, const float* __restrict__ af, int Ha,
                          const long long* __restrict__ labels, int B, const float* __restrict__ W,
                          float* __restrict__ dW, int accumulate, float* __restrict__ loss_out,
                          float* __restrict__ probs) {
  extern __shared__ float dyn[];  // [nw][2][F] per-warp gradient partials, then [nw] loss partials
  const int F = Ht + Ha;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = LOSS_THREADS / 32;
  float* lpart = dyn + (size_t)nw * 2 * F;
  // lane owns feature columns lane, lane+32, ... of the concatenated [text | audio] vector
  float g0[LOSS_CPL], g1[LOSS_CPL];
#pragma unroll
  for (int c = 0; c < LOSS_CPL; ++c) g0[c] = g1[c] = 0.f;
  float lsum = 0.f;
  const float invB = 1.f / (float)B;
  for (int b = warp; b < B; b += nw) {
    float pt0 = 0.f, pt1 = 0.f, pa0 = 0.f, pa1 = 0.f;
    float f[LOSS_CPL];
#pragma unroll
    for (int c = 0; c < LOSS_CPL; ++c) {
      const int j = c * 32 + lane;
      float v = 0.f;
      if (j < Ht) {
        v = tf[(size_t)b * Ht + j];
        pt0 = fmaf(v, W[j], pt0);
        pt1 = fmaf(v, W[F + j], pt1);
      } else if (j < F) {
        v = af[(size_t)b * Ha + (j - Ht)];
        pa0 = fmaf(v, W[j], pa0);
        pa1 = fmaf(v, W[F + j], pa1);
      }
      f[c] = v;
    }
    pt0 = warp_sum(pt0); pt1 = warp_sum(pt1); pa0 = warp_sum(pa0); pa1 = warp_sum(pa1);
    const int y = (int)labels[b];
    float m = fmaxf(pt0, pt1), e0 = expf(pt0 - m), e1 = expf(pt1 - m), z = e0 + e1;
    const float st0 = e0 / z, st1 = e1 / z;
    lsum += (m + logf(z)) - (y == 0 ? pt0 : pt1);
    m = fmaxf(pa0, pa1); e0 = expf(pa0 - m); e1 = expf(pa1 - m); z = e0 + e1;
    const float sa0 = e0 / z, sa1 = e1 / z;
    lsum += (m + logf(z)) - (y == 0 ? pa0 : pa1);
    const float dt0 = (st0 - (y == 0 ? 1.f : 0.f)) * invB, dt1 = (st1 - (y == 1 ? 1.f : 0.f)) * invB;
    const float da0 = (sa0 - (y == 0 ? 1.f : 0.f)) * invB, da1 = (sa1 - (y == 1 ? 1.f : 0.f)) * invB;
#pragma unroll
    for (int c = 0; c < LOSS_CPL; ++c) {
      const int j = c * 32 + lane;
      const bool is_t = j < Ht;
      g0[c] = fmaf(is_t ? dt0 : da0, f[c], g0[c]);
      g1[c] = fmaf(is_t ? dt1 : da1, f[c], g1[c]);
    }
    if (probs && lane == 0) {  // Softmax(fc_final(concat)) — used by the reference for accuracy only
      const float l0 = pt0 + pa0, l1 = pt1 + pa1, mm = fmaxf(l0, l1);
      const float x0 = expf(l0 - mm), x1 = expf(l1 - mm);
      probs[(size_t)b * 2 + 0] = x0 / (x0 + x1);
      probs[(size_t)b * 2 + 1] = x1 / (x0 + x1);
    }
  }
  float* gpart = dyn + (size_t)warp * 2 * F;
#pragma unroll
  for (int c = 0; c < LOSS_CPL; ++c) {
    const int j = c * 32 + lane;
    if (j < F) {
      gpart[j] = g0[c];
      gpart[F + j] = g1[c];
    }
  }
  if (lane == 0) lpart[warp] = lsum;
  __syncthreads();
  for (int i = tid; i < 2 * F; i += LOSS_THREADS) {  // fixed summation order over warps => deterministic
    float s = 0.f;
    for (int w = 0; w < nw; ++w) s += dyn[(size_t)w * 2 * F + i];
    dW[i] = accumulate ? dW[i] + s : s;
  }
  if (tid == 0) {
    float s = 0.f;
    for (int w = 0; w < nw; ++w) s += lpart[w];
    *loss_out = s * invB;
  }
}

// ---- CrossEntropyLoss applied to Softmax OUTPUTS, forward + backward in one pass -------------------------------------
// The classification scripts end their models with nn.Softmax and then feed the probabilities to nn.CrossEntropyLoss
// (audio_gru_whole.py:73, 188, 308; text_bilstm_whole.py:68, 180, 304), i.e. loss = mean_b( -log softmax(p_b)[y_b] ) with
// p = softmax(z). One warp per row: p, the row loss, and d loss / d z (chain rule through both softmaxes):
//   q = softmax(p);  g = (q - onehot(y)) / B;  dz = p * (g - sum_c p_c g_c)
constexpr int SCE_MAXC = 32;
__global__ void softmax_ce_kernel(const float* __restrict__ z, const long long* __restrict__ labels, int B, int C,
                                  float* __restrict__ probs, float* __restrict__ dz, float* __restrict__ row_loss) {
  const int lane = threadIdx.x & 31, row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B) return;
  const float NEG = -INFINITY;
  const float zv = lane < C ? z[(size_t)row * C + lane] : NEG;
  float m = warp_max(zv);
  float e = lane < C ? expf(zv - m) : 0.f;
  const float p = e / warp_sum(e);                       // model output (Softmax)
  const float pv = lane < C ? p : NEG;
  m = warp_max(pv);
  e = lane < C ? expf(pv - m) : 0.f;
  const float se = warp_sum(e);
  const float q = e / se;                                // softmax of the probabilities (inside CrossEntropyLoss)
  const long long y = labels[row];
  const float py = __shfl_sync(0xffffffffu, pv, (int)(y >= 0 && y < C ? y : 0));
  float loss = (m + logf(se)) - py;
  if (y < 0 || y >= C) loss = __int_as_float(0x7fc00000);  // a label outside [0, C) poisons the loss
  const float g = lane < C ? (q - (lane == (int)y ? 1.f : 0.f)) / (float)B : 0.f;
  const float dot = warp_sum(lane < C ? p * g : 0.f);
  if (lane < C) {
    probs[(size_t)row * C + lane] = p;
    dz[(size_t)row * C + lane] = p * (g - dot);
  }
  if (lane == 0) row_loss[row] = loss;
}
__global__ void mean_rows_kernel(const float* __restrict__ v, int n, float* __restrict__ out) {
  __shared__ float part[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += v[i];  // fixed order per thread => deterministic
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? part[threadIdx.x] : 0.f;
    s = warp_sum(s);
    if (threadIdx.x == 0) *out = s / (float)n;
  }
}

// ---- Adam (torch.optim.Adam defaults: no weight decay, no amsgrad), step counter on the device ------------------
// weight_decay is decoupled (torch.optim.AdamW: p *= 1 - lr*wd before the update; 0 gives torch.optim.Adam);
// grad_scale folds the 1/world averaging of the data-parallel all-reduce into the same pass.
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                            float* __restrict__ v, const float* __restrict__ step, size_t n, float lr, float b1,
                            float b2, float eps, float weight_decay, float grad_scale) {
  const float t = *step + 1.f;  // the increment itself is done by adam_step_kernel after this launch
  const AdamCoef c = adam_coef(t, lr, b1, b2, weight_decay);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float pi = p[i], mi = m[i], vi = v[i];
    adam_update(pi, mi, vi, g[i] * grad_scale, b1, b2, eps, c);
    m[i] = mi;
    v[i] = vi;
    p[i] = pi;
  }
}
__global__ void adam_step_kernel(float* step) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *step += 1.f;
}

}  // namespace
}  // namespace b200rnn

using namespace b200rnn;

extern "C" {

B200RNN_API int b200rnn_attention_pool(const float* seq, int64_t s_t, int64_t s_b, const float* h_n, int n_states,
                                       int B, int T, int H, const float* w_a, const float* b_a, float* ctx,
                                       void* stream_) {
  if (!seq || !h_n || !w_a || !b_a || !ctx || B < 0 || T < 1 || H < 1 || n_states < 1) {
    set_error("attention_pool: bad argument");
    return B200RNN_ERR_INVALID;
  }
  if (B == 0) return B200RNN_OK;
  // the dynamic [2H + T] floats and the kernel's static shared memory (red[2]) share the 48 KB a launch gets without
  // an opt-in; 1 KB of it is left to the static part, so that no accepted shape fails at launch
  const size_t smem = (size_t)(2 * H + T) * sizeof(float);
  if (smem > 47 * 1024) {
    set_error("attention_pool: 2*H + T = %d floats exceed the 47 KB dynamic shared-memory budget", 2 * H + T);
    return B200RNN_ERR_UNSUPPORTED;
  }
  attention_pool_kernel<<<B, 256, smem, static_cast<cudaStream_t>(stream_)>>>(seq, s_t, s_b, h_n, n_states, B, T, H, w_a,
                                                                             b_a, ctx);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

B200RNN_API int b200rnn_attention_pool_bwd(const float* seq, int64_t s_t, int64_t s_b, const float* h_n, int n_states,
                                           int B, int T, int H, const float* w_a, const float* b_a, const float* dctx,
                                           float* dseq, int64_t d_t, int64_t d_b, float* dh_n, float* dqpre,
                                           float* hsum, void* stream_) {
  if (!seq || !h_n || !w_a || !b_a || !dctx || !dseq || !dh_n || B < 0 || T < 1 || H < 1 || n_states < 1) {
    set_error("attention_pool_bwd: bad argument");
    return B200RNN_ERR_INVALID;
  }
  if (B == 0) return B200RNN_OK;
  const size_t smem = ((size_t)4 * H + 2 * T + (size_t)T * H) * sizeof(float);
  if (smem > 200 * 1024) {
    set_error("attention_pool_bwd: T*H = %d floats exceed the shared-memory budget of one CTA", T * H);
    return B200RNN_ERR_UNSUPPORTED;
  }
  static bool attr[MAX_DEVICES] = {false};
  if (!attr[current_device()]) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(attention_pool_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr[current_device()] = true;
  }
  attention_pool_bwd_kernel<<<B, 256, smem, static_cast<cudaStream_t>(stream_)>>>(seq, s_t, s_b, h_n, n_states, B, T, H, w_a,
                                                                                 b_a, dctx, dseq, d_t, d_b, dh_n, dqpre, hsum);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

B200RNN_API int b200rnn_mlp_dropout(const float* x, int B, int n, const float* W, const float* bias, float* out,
                                    int training, float p, const uint64_t* rng_hdr, uint32_t stream_id,
                                    void* stream_) {
  if (!x || !W || !bias || !out || B < 0 || n < 1 || (training && p > 0.f && !rng_hdr)) {
    set_error("mlp_dropout: bad argument");
    return B200RNN_ERR_INVALID;
  }
  if (B == 0) return B200RNN_OK;
  const size_t smem = (size_t)(MLP_TI + MLP_TB) * (n + 1) * sizeof(float);
  if (smem > 200 * 1024) {
    set_error("mlp_dropout: width %d too large", n);
    return B200RNN_ERR_UNSUPPORTED;
  }
  static bool attr[MAX_DEVICES] = {false};
  if (!attr[current_device()]) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(mlp_dropout_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr[current_device()] = true;
  }
  dim3 grid((n + MLP_TI - 1) / MLP_TI, (B + MLP_TB - 1) / MLP_TB);
  mlp_dropout_kernel<<<grid, 256, smem, static_cast<cudaStream_t>(stream_)>>>(x, B, n, W, bias, out, training, p, rng_hdr,
                                                                          stream_id);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

B200RNN_API int b200rnn_fuse_loss_grad(const float* text_feature, int Ht, const float* audio_feature, int Ha,
                                       const int64_t* labels, int B, const float* W, float* dW, int accumulate,
                                       float* loss, float* probs, void* stream_) {
  if (!text_feature || !audio_feature || !labels || !W || !dW || !loss || B < 1 || Ht < 1 || Ha < 1) {
    set_error("fuse_loss_grad: bad argument");
    return B200RNN_ERR_INVALID;
  }
  const int F = Ht + Ha;
  const size_t smem = ((size_t)(LOSS_THREADS / 32) * 2 * F + LOSS_THREADS / 32) * sizeof(float);
  if (F > LOSS_MAXF || smem > 200 * 1024) {
    set_error("fuse_loss_grad: feature width %d too large", F);
    return B200RNN_ERR_UNSUPPORTED;
  }
  static bool attr[MAX_DEVICES] = {false};
  if (!attr[current_device()]) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(fuse_loss_grad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr[current_device()] = true;
  }
  fuse_loss_grad_kernel<<<1, LOSS_THREADS, smem, static_cast<cudaStream_t>(stream_)>>>(
      text_feature, Ht, audio_feature, Ha, reinterpret_cast<const long long*>(labels), B, W, dW, accumulate, loss, probs);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

B200RNN_API int b200rnn_softmax_ce(const float* logits, const int64_t* labels, int B, int C, float* probs, float* dlogits,
                                   float* row_loss, float* loss, void* stream_) {
  if (!logits || !labels || !probs || !dlogits || !row_loss || !loss || B < 1 || C < 1) {
    set_error("softmax_ce: bad argument");
    return B200RNN_ERR_INVALID;
  }
  if (C > SCE_MAXC) {
    set_error("softmax_ce: %d classes > %d unsupported", C, SCE_MAXC);
    return B200RNN_ERR_UNSUPPORTED;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  softmax_ce_kernel<<<(B + 7) / 8, 256, 0, st>>>(logits, reinterpret_cast<const long long*>(labels), B, C, probs, dlogits,
                                               row_loss);
  B200_CUDA_CHECK(cudaGetLastError());
  mean_rows_kernel<<<1, 256, 0, st>>>(row_loss, B, loss);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch(2);
  return B200RNN_OK;
}

B200RNN_API int b200rnn_rng_next(uint64_t* hdr, uint64_t* rng_state, uint64_t consume, void* stream_) {
  if (!hdr || !rng_state) {
    set_error("rng_next: null pointer");
    return B200RNN_ERR_INVALID;
  }
  return launch_rng_setup(hdr, 0, 0, rng_state, consume, static_cast<cudaStream_t>(stream_));
}

B200RNN_API int b200rnn_adamw(float* p, const float* g, float* m, float* v, float* step, size_t n, float lr,
                              float beta1, float beta2, float eps, float weight_decay, float grad_scale,
                              int advance_step, void* stream_) {
  if (!p || !g || !m || !v || !step) {
    set_error("adamw: null pointer");
    return B200RNN_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (n > 0) {
    int blocks = (int)((n + 255) / 256);
    if (blocks > NUM_SMS * 8) blocks = NUM_SMS * 8;
    adam_kernel<<<blocks, 256, 0, st>>>(p, g, m, v, step, n, lr, beta1, beta2, eps, weight_decay, grad_scale);
    B200_CUDA_CHECK(cudaGetLastError());
    count_launch();
  }
  if (advance_step) {  // several parameter groups share one step counter: advance it after the last group
    adam_step_kernel<<<1, 32, 0, st>>>(step);
    B200_CUDA_CHECK(cudaGetLastError());
    count_launch();
  }
  return B200RNN_OK;
}

B200RNN_API int b200rnn_adam(float* p, const float* g, float* m, float* v, float* step, size_t n, float lr, float beta1,
                             float beta2, float eps, void* stream_) {
  return b200rnn_adamw(p, g, m, v, step, n, lr, beta1, beta2, eps, 0.f, 1.f, 1, stream_);
}

}  // extern "C"
