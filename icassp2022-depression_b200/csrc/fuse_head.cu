// fuse_head.cu — everything of the fuse step that comes after the two encoders, as ONE kernel:
//
//   attention_net_with_w -> fc_out (Dropout-Linear-ReLU-Dropout)        text_feature   fuse_net_whole.py:310-334, 354-355
//   fc_audio (Dropout-Linear-ReLU-Dropout) on the time-summed GRU output audio_feature  fuse_net_whole.py:362-363
//   Softmax(fc_final(cat)) | ReLU(fc_final(sigmoid(modal_attn x) * x))  model output   :368-374 | fuse_net.py:345-351
//   MyLoss: two-head CE | two-head SmoothL1 on the halves of fc_final.0.weight          :380-395 | fuse_net.py:357-366
//   d loss / d fc_final.0.weight (the only trainable tensor, :590-593)
//   [data parallel] sum of that gradient over the ranks: one-shot NVLink exchange, peer stores + flags (below)
//   torch.optim.Adam step on fc_final.0.weight                                          :416, 456
//
// Split head (classification, args.halves): the text launch also writes each row's text logit halves and text feature
// columns, an audio launch on the audio stream right after the GRU does the same for the audio half, and only the loss,
// dW, the exchange and Adam are left for one single-CTA launch after the join (fuse_loss_kernel). Every sum keeps its
// order, so the split step computes bit-identical logits, loss and update.
//
// As separate kernels this is 7 launches (attention_pool, rng_next, 2x mlp_dropout, fuse_loss_grad, adam, adam_step)
// plus a 3 KB ncclAllReduce and a 1/world scaling launch between the loss and Adam, all latency-bound. Here a CTA owns
// ROWS batch rows from the LSTM output to its rows' loss and gradient contribution; the last CTA to finish (ticket counter) reduces the
// contributions in a fixed order, exchanges the 768-float gradient with the peer GPUs, and applies Adam.
//
// Peer exchange (world > 1): every rank owns a small receive buffer (b200rnn_comm_create) that its peers map through
// CUDA IPC. Step s, parity p = s & 1: rank r stores its gradient into slot [p][r] of EVERY rank's buffer (plain
// st.global over NVLink, self included), fences at system scope and then release-stores s+1 into flag [p][r] there;
// it then acquire-polls its own flags [p][*] until all read s+1 and adds the world slots in rank order - the same
// order on every rank, so all replicas apply bit-identical updates. Two parities suffice: a rank can only re-use
// parity p at step s+2 after it finished step s+1, which needed every peer's step-(s+1) data, which a peer sends only
// after it has consumed step s. Waits are bounded (trap after ~2 s) so a protocol bug is a CUDA error, not a hung GPU.
#include <string.h>

#include "common.cuh"
#include "misc_kernels.cuh"

namespace b200rnn {

namespace {

constexpr int HEAD_THREADS = 256;
constexpr int HEAD_ROWS = 1;        // batch rows per CTA: B CTAs, the chip is covered at B = 128 (latency-bound work)
constexpr int LOSS_THREADS = 512;   // split head, loss launch: one thread per dW column up to F = 512
constexpr int ROWSTAT = 8;          // floats per batch row handed to the last CTA: dt[2], da[2], row loss (padded)
constexpr int COMM_MAX_WORLD = B200RNN_COMM_MAX_WORLD;
constexpr int COMM_PAYLOAD = 1024;  // floats per slot (fc_final.0.weight is 2 x 384 = 768; + loss)
constexpr size_t COMM_FLAG_OFF = 0;                 // uint32 flags[2][MAX_WORLD]
constexpr size_t COMM_DATA_OFF = 4096;              // float slots[2][MAX_WORLD][COMM_PAYLOAD]
constexpr size_t COMM_BYTES = COMM_DATA_OFF + (size_t)2 * COMM_MAX_WORLD * COMM_PAYLOAD * sizeof(float);

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

// keep-mask of element idx of dropout stream stream_id: same Philox layout as dropout_kernel / mlp_dropout_kernel
__device__ __forceinline__ float keep_scale(uint64_t seed, uint64_t offset, uint32_t stream_id, size_t idx,
                                            uint32_t thr, float scale) {
  Philox4 r = philox4x32_10(seed, offset + (idx >> 2), (uint64_t)stream_id);
  const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
  return rr[idx & 3] >= thr ? scale : 0.f;
}

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// ys[r][i] = act(bias[i] + sum_j W[i][j] xs[r][j]) for i in [0, n_out), r in [0, R): one warp per output row, the row
// read once with coalesced 16-byte loads and used for all R input vectors; UNR rows in flight per warp (L2 latency).
// xs / ys live in shared memory with leading dimensions ldx / ldy. Requires n % 4 == 0 and 16-byte aligned rows.
template <int R, bool RELU>
__device__ __forceinline__ void matvec_rows(const float* __restrict__ W, const float* __restrict__ bias,
                                            const float* xs, int ldx, float* ys, int ldy, int n_out, int n, int warp,
                                            int nwarps, int lane) {
  constexpr int UNR = 8;
  for (int i0 = warp * UNR; i0 < n_out; i0 += nwarps * UNR) {
    float acc[UNR][R];
#pragma unroll
    for (int u = 0; u < UNR; ++u)
#pragma unroll
      for (int r = 0; r < R; ++r) acc[u][r] = 0.f;
    for (int j = lane * 4; j < n; j += 128) {
      float4 wv[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u)
        wv[u] = (i0 + u < n_out) ? __ldg(reinterpret_cast<const float4*>(W + (size_t)(i0 + u) * n + j))
                                 : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float4 xv = *reinterpret_cast<const float4*>(xs + r * ldx + j);
#pragma unroll
        for (int u = 0; u < UNR; ++u) {
          float a = acc[u][r];
          a = fmaf(wv[u].x, xv.x, a);
          a = fmaf(wv[u].y, xv.y, a);
          a = fmaf(wv[u].z, xv.z, a);
          a = fmaf(wv[u].w, xv.w, a);
          acc[u][r] = a;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < UNR; ++u)
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float s = warp_sum(acc[u][r]);
        if (lane == 0 && i0 + u < n_out) {
          const float v = s + (bias ? bias[i0 + u] : 0.f);
          ys[r * ldy + i0 + u] = RELU ? fmaxf(v, 0.f) : v;
        }
      }
  }
}

// two-head cross entropy of one row from its logit halves pt (text) and pa (audio): d loss / d logits and the row loss
__device__ __forceinline__ float ce_row(const float pt[2], const float pa[2], long long y, float invB, float dt[2],
                                        float da[2]) {
  float lrow = 0.f;
  float m = fmaxf(pt[0], pt[1]), e0 = expf(pt[0] - m), e1 = expf(pt[1] - m), z = e0 + e1;
  lrow += (m + logf(z)) - (y == 0 ? pt[0] : pt[1]);
  dt[0] = (e0 / z - (y == 0 ? 1.f : 0.f)) * invB;
  dt[1] = (e1 / z - (y == 1 ? 1.f : 0.f)) * invB;
  m = fmaxf(pa[0], pa[1]); e0 = expf(pa[0] - m); e1 = expf(pa[1] - m); z = e0 + e1;
  lrow += (m + logf(z)) - (y == 0 ? pa[0] : pa[1]);
  da[0] = (e0 / z - (y == 0 ? 1.f : 0.f)) * invB;
  da[1] = (e1 / z - (y == 1 ? 1.f : 0.f)) * invB;
  if (y != 0 && y != 1) lrow = __int_as_float(0x7fc00000);  // a label outside {0,1} poisons the loss (NaN)
  return lrow;
}

// Softmax(fc_final(concat)) of one row - accuracy only in the reference
__device__ __forceinline__ void softmax_row(const float pt[2], const float pa[2], float* out_row) {
  const float l0 = pt[0] + pa[0], l1 = pt[1] + pa[1], mm = fmaxf(l0, l1);
  const float x0 = expf(l0 - mm), x1 = expf(l1 - mm);
  out_row[0] = x0 / (x0 + x1);
  out_row[1] = x1 / (x0 + x1);
}

// ---- one-shot peer exchange, two halves (see the file header) -------------------------------------------------------
// send: g[0..n) -> slot [parity][rank] of every rank's buffer, then the step tag into flag [parity][rank] there
__device__ __forceinline__ void peer_send(const b200rnn_fuse_head_args& a, const float* g, int n, uint32_t step, int tid,
                                          int nt) {
  const uint32_t par = step & 1u, tag = step + 1u;
  for (int idx = tid; idx < a.world * n; idx += nt) {
    const int dst = idx / n, i = idx - dst * n;
    float* slot = reinterpret_cast<float*>(static_cast<unsigned char*>(a.comm_buf[dst]) + COMM_DATA_OFF) +
                  ((size_t)par * COMM_MAX_WORLD + a.rank) * COMM_PAYLOAD;
    slot[i] = g[i];
  }
  __threadfence_system();
  __syncthreads();
  if (tid < a.world) {
    uint32_t* f = reinterpret_cast<uint32_t*>(static_cast<unsigned char*>(a.comm_buf[tid]) + COMM_FLAG_OFF) +
                  par * COMM_MAX_WORLD + a.rank;
    st_release_sys(f, tag);
  }
}
// wait for every peer's slot of `step`, then out[i] = sum over ranks in rank order (identical on every rank)
__device__ __forceinline__ void peer_wait_sum(const b200rnn_fuse_head_args& a, float* out, int n, uint32_t step, int tid,
                                              int nt) {
  const uint32_t par = step & 1u, tag = step + 1u;
  if (tid < a.world) {
    const uint32_t* mine = reinterpret_cast<const uint32_t*>(static_cast<unsigned char*>(a.comm_buf[a.rank]) + COMM_FLAG_OFF) +
                           par * COMM_MAX_WORLD + tid;
    const long long t0 = clock64();
    while (ld_acquire_sys(mine) != tag) {
      if (clock64() - t0 > 4000000000ll) __trap();  // ~2 s: a peer died or the protocol is broken
    }
  }
  __syncthreads();
  const float* slots = reinterpret_cast<const float*>(static_cast<unsigned char*>(a.comm_buf[a.rank]) + COMM_DATA_OFF) +
                       (size_t)par * COMM_MAX_WORLD * COMM_PAYLOAD;
  for (int i = tid; i < n; i += nt) {
    float s = 0.f;
    for (int r = 0; r < a.world; ++r) s += __ldcv(slots + (size_t)r * COMM_PAYLOAD + i);  // rank order on every rank
    out[i] = s;
  }
  __syncthreads();
}

// Deferred half of the exchange: applies the update of the oldest step that was sent but not applied yet (if any).
__global__ void __launch_bounds__(HEAD_THREADS) fuse_head_finish_kernel(const b200rnn_fuse_head_args a) {
  __shared__ float g[COMM_PAYLOAD];
  const int tid = threadIdx.x;
  const int n = (a.regression ? 1 : 2) * (a.Ht + a.Ha);
  const uint32_t done = *a.comm_done, sent = *a.comm_step;
  if (done == sent) return;  // nothing pending (first step, or already flushed)
  peer_wait_sum(a, g, n, done, tid, HEAD_THREADS);
  const float t = *a.adam_step + 1.f;
  const AdamCoef c = adam_coef(t, a.lr, a.beta1, a.beta2, 0.f);
  for (int i = tid; i < n; i += HEAD_THREADS) {
    float w = a.W[i], mi = a.adam_m[i], vi = a.adam_v[i];
    adam_update(w, mi, vi, g[i] * a.grad_scale, a.beta1, a.beta2, a.eps, c);
    a.adam_m[i] = mi;
    a.adam_v[i] = vi;
    a.W[i] = w;
  }
  __syncthreads();
  if (tid == 0) {
    *a.adam_step = t;
    *a.comm_done = done + 1u;
  }
}

// Per-row scalars rst[B][ROWSTAT] (in shared memory) and the feature matrix feat_ws[B][F] -> dW (fixed batch order),
// the loss (fixed order), the peer exchange, the Philox offset advance and Adam. Run by all NT threads of ONE CTA.
template <int NT>
__device__ __forceinline__ void loss_tail(const b200rnn_fuse_head_args& a, const float* rst, const float* feat_ws,
                                          bool drop, uint64_t offset, int tid, int lane, int warp) {
  const int Ht = a.Ht, F = a.Ht + a.Ha, B = a.B, C = a.regression ? 1 : 2;
  for (int j = tid; j < F; j += NT) {
    float g0 = 0.f, g1 = 0.f;
    const int so = (j < Ht) ? 0 : 2;
    int b = 0;
    for (; b + 16 <= B; b += 16) {  // 16 independent coalesced loads in flight per thread, then the ordered adds
      float fv[16];
#pragma unroll
      for (int u = 0; u < 16; ++u) fv[u] = __ldcg(feat_ws + (size_t)(b + u) * F + j);
#pragma unroll
      for (int u = 0; u < 16; ++u) {
        g0 = fmaf(rst[(b + u) * ROWSTAT + so], fv[u], g0);
        g1 = fmaf(rst[(b + u) * ROWSTAT + so + 1], fv[u], g1);
      }
    }
    for (; b < B; ++b) {
      const float fv = __ldcg(feat_ws + (size_t)b * F + j);
      g0 = fmaf(rst[b * ROWSTAT + so], fv, g0);
      g1 = fmaf(rst[b * ROWSTAT + so + 1], fv, g1);
    }
    a.dw[j] = a.accumulate ? a.dw[j] + g0 : g0;
    if (C == 2) a.dw[F + j] = a.accumulate ? a.dw[F + j] + g1 : g1;
  }
  if (warp == 0) {  // loss = sum of the row losses, fixed order
    float l = 0.f;
    for (int b = lane; b < B; b += 32) l += rst[b * ROWSTAT + 4];
    l = warp_sum(l);
    if (lane == 0) a.dw[C * F] = l;
  }
  __syncthreads();
  bool apply_update = true;
  if (a.world > 1) {
    const uint32_t step = *a.comm_step;  // device-resident: a captured graph advances it at every replay
    const int NX = C * F;  // the loss stays local (each rank reports its own shard's loss, like the reference would)
    peer_send(a, a.dw, NX, step, tid, NT);
    if (a.defer_exchange) {
      apply_update = false;  // b200rnn_fuse_head_finish waits, sums and applies Adam (next step, beside the encoders)
    } else {
      peer_wait_sum(a, a.dw, NX, step, tid, NT);
    }
    if (tid == 0) *a.comm_step = step + 1u;
    __syncthreads();
  }
  if (tid == 0) {
    *a.loss = a.dw[C * F];
    *a.ticket = 0u;  // re-armed for the next launch (graph replay)
    if (drop && a.rng_state) a.rng_state[1] = offset + a.rng_consume;
  }
  if (a.do_adam && apply_update) {  // torch.optim.Adam (no weight decay, no amsgrad); grad_scale = 1/world
    const float t = *a.adam_step + 1.f;
    const AdamCoef c = adam_coef(t, a.lr, a.beta1, a.beta2, 0.f);
    for (int i = tid; i < C * F; i += NT) {
      float w = a.W[i], mi = a.adam_m[i], vi = a.adam_v[i];
      adam_update(w, mi, vi, a.dw[i] * a.grad_scale, a.beta1, a.beta2, a.eps, c);
      a.adam_m[i] = mi;
      a.adam_v[i] = vi;
      a.W[i] = w;
    }
    __syncthreads();
    if (tid == 0) *a.adam_step = t;
  }
}

__global__ void __launch_bounds__(HEAD_THREADS) fuse_head_kernel(const b200rnn_fuse_head_args a) {
  constexpr int R = HEAD_ROWS;
  extern __shared__ __align__(16) float sm[];
  const int Ht = a.Ht, Ha = a.Ha, F = Ht + Ha, T = a.T, B = a.B, C = a.regression ? 1 : 2;
  // shared-memory carve-up (floats); every row block is a multiple of 4 floats
  float* hsum = sm;                 // [R][Ht]
  float* q = hsum + R * Ht;         // [R][Ht]
  float* ctx = q + R * Ht;          // [R][Ht]   attention context, then dropout-1 applied in place
  float* feat = ctx + R * Ht;       // [R][F]    text_feature | audio_feature (after dropout-2)
  float* xa = feat + R * F;         // [R][Ha]   pooled audio with dropout-1
  float* gate = xa + R * Ha;        // [R][F]    regression: sigmoid(modal_attn x) * x
  float* score = gate + R * F;      // [R][Tpad]
  const int Tpad = (T + 3) & ~3;
  float* red = score + R * Tpad;    // [32] scratch
  float* hst = red + 32;            // [R][T][Ht] h_t = fwd + rev halves of the BiLSTM output
  __shared__ int s_last;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = HEAD_THREADS / 32;
  const int b0 = blockIdx.x * R;
  const bool text = !a.tf_in && (a.seq || a.ctx_in);  // this launch computes the text half

  // fc_audio.1.weight into L2 before the wait. The GRU before it never triggers its dependents early, so a programmatic
  // launch only overlaps this with the GRU's last CTAs draining and its memory flush, not with its steps
  if (a.pooled) {
    const size_t line = (size_t)blockIdx.x * HEAD_THREADS + tid, lines = (size_t)Ha * Ha * sizeof(float) / 128;
    if (line < lines) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.w_a + line * 32));
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");  // no-op unless launched programmatically

  float* feat_ws = a.dw_part ? a.dw_part + (size_t)B * ROWSTAT : nullptr;  // [B][F] features for the gradient pass
  const bool drop = a.training && a.p > 0.f;
  const uint32_t thr = (uint32_t)fminf(a.p * 4294967296.0f, 4294967295.0f);
  const float scale = a.p < 1.f ? 1.f / (1.f - a.p) : 0.f;
  uint64_t seed = 0, offset = 0;
  if (drop) {
    seed = a.rng_state[0];
    offset = a.rng_state[1];
  }

  // ---------------- text branch: attention pooling (text_bilstm_whole.py:74-99) ----------------------------------
  if (a.tf_in) {
    // text stage already done by an earlier launch on the text branch's stream: take its text_feature as is
    for (int idx = tid; idx < R * Ht; idx += HEAD_THREADS) {
      const int r = idx / Ht, j = idx - r * Ht, b = b0 + r;
      feat[r * F + j] = (b < B) ? a.tf_in[(size_t)b * Ht + j] : 0.f;
    }
  } else if (a.seq) {
    for (int idx = tid; idx < R * Ht; idx += HEAD_THREADS) {
      const int r = idx / Ht, j = idx - r * Ht, b = b0 + r;
      float s = 0.f;
      if (b < B)
        for (int k = 0; k < a.n_states; ++k) s += a.h_n[((size_t)k * B + b) * Ht + j];
      hsum[idx] = s;
    }
    __syncthreads();
    // h_t = seq[t,b,:Ht] + seq[t,b,Ht:] of this CTA's rows -> shared memory in ONE pass of independent, coalesced
    // loads (the scores and the context both walk over t: from global memory that was ~2T dependent round trips)
    for (int idx = tid; idx < R * T * Ht; idx += HEAD_THREADS) {
      const int r = idx / (T * Ht), rem = idx - r * (T * Ht), t = rem / Ht, j = rem - t * Ht, b = b0 + r;
      float v = 0.f;
      if (b < B) {
        const float* row = a.seq + (long long)t * a.seq_st + (long long)b * a.seq_sb;
        v = row[j] + row[Ht + j];
      }
      hst[idx] = v;
    }
    matvec_rows<R, true>(a.w_att, a.b_att, hsum, Ht, q, Ht, Ht, Ht, warp, nw, lane);  // q = ReLU(W_a hsum + b_a)
    __syncthreads();
    for (int idx = warp; idx < R * T; idx += nw) {  // scores: one warp per (row, time step)
      const int r = idx / T, t = idx - r * T;
      float s = 0.f;
      for (int j = lane; j < Ht; j += 32) s += q[r * Ht + j] * tanhf(hst[(r * T + t) * Ht + j]);
      s = warp_sum(s);
      if (lane == 0) score[r * Tpad + t] = s;
    }
    __syncthreads();
    if (warp < R) {  // softmax over T, one warp per row
      const int r = warp;
      float m = -INFINITY;
      for (int t = lane; t < T; t += 32) m = fmaxf(m, score[r * Tpad + t]);
      m = warp_max(m);
      float z = 0.f;
      for (int t = lane; t < T; t += 32) {
        const float e = expf(score[r * Tpad + t] - m);
        score[r * Tpad + t] = e;
        z += e;
      }
      z = warp_sum(z);
      if (lane == 0) red[r] = 1.f / z;
    }
    __syncthreads();
    for (int idx = tid; idx < R * Ht; idx += HEAD_THREADS) {
      const int r = idx / Ht, j = idx - r * Ht, b = b0 + r;
      float acc = 0.f;
      if (b < B) {
        for (int t = 0; t < T; ++t) acc += score[r * Tpad + t] * hst[(r * T + t) * Ht + j];
        acc *= red[r];
        if (a.ctx_out) a.ctx_out[(size_t)b * Ht + j] = acc;
        if (drop) acc *= keep_scale(seed, offset, 0, (size_t)b * Ht + j, thr, scale);  // fc_out[0] Dropout
      }
      ctx[idx] = acc;
    }
  } else if (a.ctx_in) {  // attention context given (features computed elsewhere)
    for (int idx = tid; idx < R * Ht; idx += HEAD_THREADS) {
      const int r = idx / Ht, j = idx - r * Ht, b = b0 + r;
      float v = (b < B) ? a.ctx_in[(size_t)b * Ht + j] : 0.f;
      if (drop && b < B) v *= keep_scale(seed, offset, 0, (size_t)b * Ht + j, thr, scale);
      ctx[idx] = v;
    }
  }
  // ---------------- audio branch input: time-summed GRU output with fc_audio[0] Dropout ---------------------------
  if (a.pooled)
    for (int idx = tid; idx < R * Ha; idx += HEAD_THREADS) {
      const int r = idx / Ha, j = idx - r * Ha, b = b0 + r;
      float v = (b < B) ? a.pooled[(size_t)b * Ha + j] : 0.f;
      if (drop && b < B) v *= keep_scale(seed, offset, 2, (size_t)b * Ha + j, thr, scale);
      xa[idx] = v;
    }
  __syncthreads();
  // ---------------- the two Linear+ReLU heads, then their output Dropout ------------------------------------------
  if (text) matvec_rows<R, true>(a.w_t, a.b_t, ctx, Ht, feat, F, Ht, Ht, warp, nw, lane);
  if (a.pooled) matvec_rows<R, true>(a.w_a, a.b_a, xa, Ha, feat + Ht, F, Ha, Ha, warp, nw, lane);
  __syncthreads();
  for (int idx = tid; idx < R * F; idx += HEAD_THREADS) {
    const int r = idx / F, j = idx - r * F, b = b0 + r;
    if ((j < Ht) ? !text : (a.pooled == nullptr)) continue;  // half not produced by this launch
    float v = feat[idx];
    if (b < B) {
      if (drop)
        v *= (j < Ht) ? keep_scale(seed, offset, 1, (size_t)b * Ht + j, thr, scale)
                      : keep_scale(seed, offset, 3, (size_t)b * Ha + (j - Ht), thr, scale);
      if (j < Ht) {
        if (a.text_feature) a.text_feature[(size_t)b * Ht + j] = v;
      } else {
        if (a.audio_feature) a.audio_feature[(size_t)b * Ha + (j - Ht)] = v;
      }
    } else {
      v = 0.f;
    }
    feat[idx] = v;
  }
  __syncthreads();
  if (a.halves) {  // split head: this half's logits and feature columns of the row; fuse_loss_kernel does the rest
    if (warp < R && b0 + warp < B) {
      const int r = warp, b = b0 + r;
      const float* f = feat + r * F;
      float h[2] = {0.f, 0.f};
      for (int j = lane; j < F; j += 32) {  // the lane-strided chains of the whole-row loop below, one half of them
        if ((j < Ht) != text) continue;
        const float v = f[j];
#pragma unroll
        for (int c = 0; c < 2; ++c)
          if (c < C) h[c] = fmaf(v, a.W[(size_t)c * F + j], h[c]);
      }
      h[0] = warp_sum(h[0]);
      if (C == 2) h[1] = warp_sum(h[1]);
      if (lane == 0) {
        a.halves[(size_t)b * 4 + (text ? 0 : 2)] = h[0];
        a.halves[(size_t)b * 4 + (text ? 1 : 3)] = h[1];
      }
    }
    for (int idx = tid; idx < R * F; idx += HEAD_THREADS) {
      const int r = idx / F, j = idx - r * F, b = b0 + r;
      if (b < B && (j < Ht) == text) feat_ws[(size_t)b * F + j] = feat[idx];
    }
    return;
  }
  if (!a.W) return;  // features only

  // ---------------- model output + two-head loss + per-row gradient contribution ---------------------------------
  if (a.regression && a.w_modal && a.out)  // ReLU(fc_final(sigmoid(modal_attn x) * x)), fuse_net.py:345-351
    matvec_rows<R, false>(a.w_modal, nullptr, feat, F, gate, F, F, F, warp, nw, lane);
  __syncthreads();
  const float invB = 1.f / (float)B;
  if (warp < R) {
    const int r = warp, b = b0 + r;
    if (b < B) {
      const float* f = feat + r * F;
      float pt[2] = {0.f, 0.f}, pa[2] = {0.f, 0.f}, po = 0.f;
      for (int j = lane; j < F; j += 32) {
        const float v = f[j];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          if (c < C) {
            const float w = a.W[(size_t)c * F + j];
            if (j < Ht) pt[c] = fmaf(v, w, pt[c]);
            else pa[c] = fmaf(v, w, pa[c]);
          }
        }
        if (a.regression && a.w_modal && a.out) {
          const float gt = 1.f / (1.f + expf(-gate[r * F + j]));
          po = fmaf(gt * v, a.W[j], po);
        }
      }
      pt[0] = warp_sum(pt[0]); pa[0] = warp_sum(pa[0]);
      if (C == 2) { pt[1] = warp_sum(pt[1]); pa[1] = warp_sum(pa[1]); }
      float dt[2] = {0.f, 0.f}, da[2] = {0.f, 0.f}, lrow = 0.f;
      if (!a.regression) {
        lrow = ce_row(pt, pa, reinterpret_cast<const long long*>(a.labels)[b], invB, dt, da);
        if (a.out && lane == 0) softmax_row(pt, pa, a.out + (size_t)b * 2);
      } else {  // SmoothL1 (beta = 1, mean over the B x 1 predictions), fuse_net.py:357-366
        const float y = reinterpret_cast<const float*>(a.labels)[b];
        float d = pt[0] - y;
        lrow += fabsf(d) < 1.f ? 0.5f * d * d : fabsf(d) - 0.5f;
        dt[0] = fminf(fmaxf(d, -1.f), 1.f) * invB;
        d = pa[0] - y;
        lrow += fabsf(d) < 1.f ? 0.5f * d * d : fabsf(d) - 0.5f;
        da[0] = fminf(fmaxf(d, -1.f), 1.f) * invB;
        if (a.out) {
          po = warp_sum(po);
          if (lane == 0) a.out[b] = a.w_modal ? fmaxf(po, 0.f) : fmaxf(pt[0] + pa[0], 0.f);
        }
      }
      if (lane == 0) {  // what the last CTA needs from this row: the four logit gradients and the row's loss
        float* st = a.dw_part + (size_t)b * ROWSTAT;
        st[0] = dt[0]; st[1] = dt[1]; st[2] = da[0]; st[3] = da[1]; st[4] = lrow * invB;
      }
    }
  }
  // the features of this CTA's rows, for the gradient pass of the last CTA (dW = d^T [tf | af])
  for (int idx = tid; idx < R * F; idx += HEAD_THREADS) {
    const int r = idx / F, j = idx - r * F, b = b0 + r;
    if (b < B) feat_ws[(size_t)b * F + j] = feat[idx];
  }

  // ---------------- last CTA: deterministic reduction over the batch, peer exchange, Adam --------------------------
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = (atomicAdd(a.ticket, 1u) == gridDim.x - 1) ? 1 : 0;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // dW[c][j] = sum_b d[b][c] * f[b][j]: a [C x B] x [B x F] product. Thread j walks the batch in a fixed order
  // (deterministic), every load is a coalesced row segment of the feature matrix; the 5 per-row scalars sit in shared
  // memory (the feature staging area of this CTA is free now).
  float* rst = sm;  // [B][ROWSTAT] : B * 8 floats <= the R*(3Ht+2F+Ha+T) floats carved above? checked on the host
  for (int idx = tid; idx < B * ROWSTAT; idx += HEAD_THREADS) rst[idx] = __ldcg(a.dw_part + idx);
  __syncthreads();
  loss_tail<HEAD_THREADS>(a, rst, feat_ws, drop, offset, tid, lane, warp);
}

// Split head, after the join: the loss of every row from the halves the two branch launches wrote, then loss_tail.
// One CTA: one thread per row, then the same fixed-order reductions as the last CTA of fuse_head_kernel, with one
// thread per dW column.
__global__ void __launch_bounds__(LOSS_THREADS) fuse_loss_kernel(const b200rnn_fuse_head_args a) {
  extern __shared__ __align__(16) float rst[];  // [B][ROWSTAT]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, B = a.B;
  const float invB = 1.f / (float)B;
  const bool drop = a.training && a.p > 0.f;
  const uint64_t offset = drop ? a.rng_state[1] : 0;
  for (int b = tid; b < B; b += LOSS_THREADS) {
    const float4 h = __ldcg(reinterpret_cast<const float4*>(a.halves) + b);
    const float pt[2] = {h.x, h.y}, pa[2] = {h.z, h.w};
    float dt[2], da[2];
    const float lrow = ce_row(pt, pa, reinterpret_cast<const long long*>(a.labels)[b], invB, dt, da);
    if (a.out) softmax_row(pt, pa, a.out + (size_t)b * 2);
    float* st = rst + b * ROWSTAT;
    st[0] = dt[0]; st[1] = dt[1]; st[2] = da[0]; st[3] = da[1]; st[4] = lrow * invB;
  }
  __syncthreads();
  loss_tail<LOSS_THREADS>(a, rst, a.dw_part + (size_t)B * ROWSTAT, drop, offset, tid, lane, warp);
}

size_t head_smem_floats(int B, int Ht, int Ha, int T, bool loss_stage) {
  const int F = Ht + Ha, Tpad = (T + 3) & ~3;
  size_t n = (size_t)HEAD_ROWS * (3 * Ht + 2 * F + Ha + Tpad + (size_t)T * Ht) + 32;
  const size_t rst = loss_stage ? (size_t)B * ROWSTAT : 0;  // the last CTA re-uses the area for the per-row scalars
  return n > rst ? n : rst;
}

}  // namespace
}  // namespace b200rnn

using namespace b200rnn;

extern "C" {

B200RNN_API size_t b200rnn_fuse_head_scratch_floats(int B, int Ht, int Ha, int regression) {
  (void)regression;
  return (size_t)(B > 0 ? B : 0) * (size_t)(ROWSTAT + Ht + Ha);  // per-row scalars, then the feature matrix [B, F]
}

B200RNN_API int b200rnn_fuse_head(const b200rnn_fuse_head_args* args, void* stream_) {
  if (!args || args->struct_bytes != sizeof(b200rnn_fuse_head_args)) {
    set_error("fuse_head: null or mismatched argument block (%u bytes passed, library expects %zu)",
              args ? args->struct_bytes : 0u, sizeof(b200rnn_fuse_head_args));
    return B200RNN_ERR_INVALID;
  }
  const b200rnn_fuse_head_args& a = *args;
  if (a.B < 0 || a.Ht < 4 || a.Ha < 4 || a.Ht % 4 || a.Ha % 4) {
    set_error("fuse_head: unsupported widths Ht=%d Ha=%d (multiples of 4)", a.Ht, a.Ha);
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (a.B == 0) return B200RNN_OK;
  const bool text_in = a.tf_in || a.seq || a.ctx_in;
  const bool have_text = a.tf_in ? true
                         : (a.seq ? (a.h_n && a.w_att && a.b_att && a.T >= 1 && a.n_states >= 1) : (a.ctx_in != nullptr));
  // split head: one branch per launch (its halves), or neither (the loss launch)
  const bool loss_launch = a.halves && !text_in && !a.pooled;
  if (a.halves && (a.regression || !a.W || !a.dw_part || (text_in && a.pooled) ||
                   (reinterpret_cast<uintptr_t>(a.halves) & 15u))) {
    set_error("fuse_head: halves: classification only, 16-byte aligned, needs W and dw_part, and one branch (or none) "
              "per launch");
    return B200RNN_ERR_INVALID;
  }
  const bool branch_ok = a.halves ? (loss_launch || a.pooled || (have_text && !a.tf_in)) : have_text;
  if (!branch_ok || (text_in && !a.tf_in && (!a.w_t || !a.b_t)) || (a.pooled && (!a.w_a || !a.b_a)) ||
      (!a.pooled && a.W && !a.halves)) {
    set_error("fuse_head: null pointer argument (or the loss stage without the audio stage)");
    return B200RNN_ERR_INVALID;
  }
  if (a.training && a.p > 0.f && !a.rng_state) {
    set_error("fuse_head: train-mode dropout needs rng_state");
    return B200RNN_ERR_INVALID;
  }
  if (a.W && (!a.halves || loss_launch)) {
    if (!a.labels || !a.dw_part || !a.dw || !a.loss || !a.ticket) {
      set_error("fuse_head: loss stage needs labels, dw_part, dw, loss and ticket");
      return B200RNN_ERR_INVALID;
    }
    if (a.do_adam && (!a.adam_m || !a.adam_v || !a.adam_step)) {
      set_error("fuse_head: Adam stage needs m, v and step");
      return B200RNN_ERR_INVALID;
    }
    const int C = a.regression ? 1 : 2;
    if (a.world > 1) {
      if (a.world > COMM_MAX_WORLD || a.rank < 0 || a.rank >= a.world || !a.comm_step ||
          C * (a.Ht + a.Ha) > COMM_PAYLOAD || (a.defer_exchange && !a.comm_done)) {
        set_error("fuse_head: bad peer-exchange arguments (world=%d rank=%d)", a.world, a.rank);
        return B200RNN_ERR_INVALID;
      }
      for (int r = 0; r < a.world; ++r)
        if (!a.comm_buf[r]) {
          set_error("fuse_head: peer buffer %d is not mapped", r);
          return B200RNN_ERR_INVALID;
        }
    }
  }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (loss_launch) {
    const size_t smem = (size_t)a.B * ROWSTAT * sizeof(float);
    if (smem > 200 * 1024) {
      set_error("fuse_head: batch too large for the single-CTA loss launch");
      return B200RNN_ERR_UNSUPPORTED;
    }
    static bool loss_attr[MAX_DEVICES] = {false};
    if (!loss_attr[current_device()]) {
      B200_CUDA_CHECK(cudaFuncSetAttribute(fuse_loss_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
      loss_attr[current_device()] = true;
    }
    fuse_loss_kernel<<<1, LOSS_THREADS, smem, stream>>>(a);
    B200_CUDA_CHECK(cudaGetLastError());
    count_launch();
    return B200RNN_OK;
  }
  const bool stage_only = a.halves || !a.W;
  const size_t smem = head_smem_floats(a.B, a.Ht, a.Ha, (a.seq && !a.tf_in) ? a.T : 0, !stage_only) * sizeof(float);
  if (smem > 200 * 1024) {
    set_error("fuse_head: widths too large for one CTA");
    return B200RNN_ERR_UNSUPPORTED;
  }
  static bool attr[MAX_DEVICES] = {false};
  if (!attr[current_device()]) {
    B200_CUDA_CHECK(cudaFuncSetAttribute(fuse_head_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr[current_device()] = true;
  }
  const int grid = (a.B + HEAD_ROWS - 1) / HEAD_ROWS;
  if (a.halves && a.pooled) {
    // the audio launch follows the GRU on its stream: launched programmatically, its CTAs start (and prefetch
    // fc_audio.1.weight) as the recurrence's CTAs exit; griddepcontrol.wait holds every read of the GRU's output
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(HEAD_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr1[1];
    attr1[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr1[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr1;
    cfg.numAttrs = 1;
    B200_CUDA_CHECK(cudaLaunchKernelEx(&cfg, fuse_head_kernel, a));
  } else {
    fuse_head_kernel<<<grid, HEAD_THREADS, smem, stream>>>(a);
  }
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

B200RNN_API int b200rnn_fuse_head_finish(const b200rnn_fuse_head_args* args, void* stream_) {
  if (!args || args->struct_bytes != sizeof(b200rnn_fuse_head_args)) {
    set_error("fuse_head_finish: null or mismatched argument block");
    return B200RNN_ERR_INVALID;
  }
  const b200rnn_fuse_head_args& a = *args;
  if (a.world <= 1) return B200RNN_OK;  // nothing is ever deferred without peers
  const int C = a.regression ? 1 : 2;
  if (a.world > COMM_MAX_WORLD || a.rank < 0 || a.rank >= a.world || !a.comm_step || !a.comm_done || !a.W || !a.adam_m ||
      !a.adam_v || !a.adam_step || C * (a.Ht + a.Ha) > COMM_PAYLOAD) {
    set_error("fuse_head_finish: bad argument");
    return B200RNN_ERR_INVALID;
  }
  for (int r = 0; r < a.world; ++r)
    if (!a.comm_buf[r]) {
      set_error("fuse_head_finish: peer buffer %d is not mapped", r);
      return B200RNN_ERR_INVALID;
    }
  fuse_head_finish_kernel<<<1, HEAD_THREADS, 0, static_cast<cudaStream_t>(stream_)>>>(a);
  B200_CUDA_CHECK(cudaGetLastError());
  count_launch();
  return B200RNN_OK;
}

/* ---- peer exchange buffers (setup path, not the hot path) ------------------------------------------------------ */
B200RNN_API size_t b200rnn_comm_bytes(void) { return COMM_BYTES; }

B200RNN_API int b200rnn_comm_create(void** local_buf, unsigned char* ipc_handle_out) {
  if (!local_buf || !ipc_handle_out) {
    set_error("comm_create: null pointer");
    return B200RNN_ERR_INVALID;
  }
  static_assert(sizeof(cudaIpcMemHandle_t) == B200RNN_IPC_HANDLE_BYTES, "IPC handle size");
  void* p = nullptr;
  B200_CUDA_CHECK(cudaMalloc(&p, COMM_BYTES));
  B200_CUDA_CHECK(cudaMemset(p, 0, COMM_BYTES));
  B200_CUDA_CHECK(cudaDeviceSynchronize());
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    cudaFree(p);
    set_error("comm_create: cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
    cudaGetLastError();
    return B200RNN_ERR_CUDA;
  }
  memcpy(ipc_handle_out, &h, sizeof(h));
  *local_buf = p;
  return B200RNN_OK;
}

B200RNN_API int b200rnn_comm_open(const unsigned char* ipc_handle, void** peer_buf) {
  if (!ipc_handle || !peer_buf) {
    set_error("comm_open: null pointer");
    return B200RNN_ERR_INVALID;
  }
  cudaIpcMemHandle_t h;
  memcpy(&h, ipc_handle, sizeof(h));
  void* p = nullptr;
  cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) {
    set_error("comm_open: cudaIpcOpenMemHandle failed: %s (peer access over NVLink/PCIe is required)",
              cudaGetErrorString(e));
    cudaGetLastError();
    return B200RNN_ERR_CUDA;
  }
  *peer_buf = p;
  return B200RNN_OK;
}

B200RNN_API int b200rnn_comm_close(void* peer_buf) {
  if (peer_buf) B200_CUDA_CHECK(cudaIpcCloseMemHandle(peer_buf));
  return B200RNN_OK;
}

B200RNN_API int b200rnn_comm_destroy(void* local_buf) {
  if (local_buf) B200_CUDA_CHECK(cudaFree(local_buf));
  return B200RNN_OK;
}

}  // extern "C"
