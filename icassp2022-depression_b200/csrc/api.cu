// api.cu — the C ABI (include/b200rnn.h) and the host-side sequencing of one multi-layer GRU / (Bi)LSTM
// forward or backward pass. Everything is enqueued on the caller's stream; no allocation, no sync.
//
// Per layer, forward:   [K1 GEMM per direction]  ->  [one persistent recurrence launch, all directions]
//                       -> [K7 dropout, train mode, not after the last layer]
// Per layer, backward:  [W_hh transpose per direction] -> [one persistent BPTT launch, all directions]
//                       -> [bias reduce, wgrad GEMMs (split-K, deterministic), dgrad GEMM]
#include <atomic>
#include <mutex>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "cell_kernels.cuh"
#include "gemm_f32.cuh"
#include "gemm_h16_layout.cuh"
#include "h16.cuh"
#include "misc_kernels.cuh"
#include "rnn_kernels.cuh"

namespace b200rnn {

static thread_local char g_err[512] = {0};
static std::atomic<unsigned long long> g_launches{0};
long long* g_trace = nullptr;  // debug hook: device buffer [T][8] for rec_fwd phase timestamps

void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

namespace {

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// proj_size of a descriptor: the field exists only when B200RNN_FLAG_PROJ says so (a descriptor may end at `flags`)
inline int desc_proj(const b200rnn_desc* d) { return (d->flags & B200RNN_FLAG_PROJ) ? d->proj_size : 0; }
// the model count, read only under B200RNN_FLAG_MODELS
inline int desc_models(const b200rnn_desc* d) { return (d->flags & B200RNN_FLAG_MODELS) ? d->models : 1; }

// The model-shell entry points (b200rnn_forward_fused, _backward_fused, _prepare_weights, _wcache_bytes) run only the
// GRU / LSTM at the fixed hidden sizes 128 and 256: their fusions (LayerNorm prologue, pooling, weight cache, the
// fp16-pair no-grad recurrence) are built for those
int check_shell_desc(const b200rnn_desc* d, const char* what) {
  if (d && desc_models(d) != 1) {
    set_error("%s: the model-shell entry points run one model (use the _hx entry points for several)", what);
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (d && (d->flags & (B200RNN_FLAG_F16 | B200RNN_FLAG_BF16 | B200RNN_FLAG_F32_PARAMS))) {
    set_error("%s: the model-shell entry points and the weight cache are float32 only (use the _hx entry points for "
              "16-bit tensors)", what);
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (d && is_elman(d->mode)) {
    set_error("%s: the model-shell entry points take the GRU and the LSTM (got mode %d; use the _hx entry points)",
              what, d->mode);
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (d && d->hidden_size != 128 && d->hidden_size != 256) {
    set_error("%s: the model-shell entry points take hidden_size 128 and 256 (got %d; use the _hx entry points)", what,
              d->hidden_size);
    return B200RNN_ERR_UNSUPPORTED;
  }
  return B200RNN_OK;
}

struct Dims {
  int mode, B, T, I, H, L, D, G;
  int P, HO, NPAR;  // proj_size (0: none), width of h / the layer output per direction, parameters per (layer, dir)
  size_t TB, GH, DH;  // DH = D * HO: width of a layer's output
  bool training;
  float p;
  int dt;  // DT_F32, or DT_F16 / DT_BF16: the caller's tensors are 16-bit (B200RNN_FLAG_F16 / _BF16)
  bool master;  // B200RNN_FLAG_F32_PARAMS: the parameters and their gradients are fp32 (the rest is 16-bit)
  int M;        // models (B200RNN_FLAG_MODELS), 1 without the flag
  const int64_t* ms;  // with M > 1: the caller's model strides (x, rng_state, params[i])
};

int check_desc(const b200rnn_desc* d, Dims* o) {
  if (!d) {
    set_error("null descriptor");
    return B200RNN_ERR_INVALID;
  }
  if (d->mode != B200RNN_GRU && d->mode != B200RNN_LSTM && !is_elman(d->mode)) {
    set_error("mode must be B200RNN_GRU, B200RNN_LSTM, B200RNN_RNN_TANH or B200RNN_RNN_RELU (got %d)", d->mode);
    return B200RNN_ERR_INVALID;
  }
  if (d->batch < 0 || d->seq_len < 0 || d->input_size <= 0 || d->num_layers <= 0 ||
      (d->num_dirs != 1 && d->num_dirs != 2)) {
    set_error("bad shape: B=%d T=%d I=%d L=%d D=%d", d->batch, d->seq_len, d->input_size, d->num_layers,
              d->num_dirs);
    return B200RNN_ERR_INVALID;
  }
  // GRU / LSTM 128 and 256 run the fixed configs of rnn_rec.cu, every other multiple of 16 up to 1024 the runtime-sized
  // kernels of rnn_anyh.cu; the Elman modes run those at every one of them
  if (!anyh_hidden_size(d->hidden_size)) {
    set_error("hidden_size %d unsupported: the sm_90a recurrence kernels take multiples of 16 from 16 to 1024",
              d->hidden_size);
    return B200RNN_ERR_UNSUPPORTED;
  }
  const int P = desc_proj(d);
  if (P < 0 || (P > 0 && (d->mode != B200RNN_LSTM || P >= d->hidden_size))) {
    set_error("proj_size %d invalid: an LSTM takes 0 <= proj_size < hidden_size, a GRU none", P);
    return B200RNN_ERR_INVALID;
  }
  if (P > 0 && ((d->hidden_size != 128 && d->hidden_size != 256) ||
                (P != d->hidden_size / 4 && P != d->hidden_size / 2))) {
    set_error("proj_size %d unsupported: the projected kernels are built for hidden_size 128 and 256 with "
              "proj_size hidden_size/4 and hidden_size/2", P);
    return B200RNN_ERR_UNSUPPORTED;
  }
  const uint32_t h16 = d->flags & (B200RNN_FLAG_F16 | B200RNN_FLAG_BF16);
  if (h16 == (B200RNN_FLAG_F16 | B200RNN_FLAG_BF16)) {
    set_error("B200RNN_FLAG_F16 and B200RNN_FLAG_BF16 exclude each other");
    return B200RNN_ERR_UNSUPPORTED;
  }
  const bool master = (d->flags & B200RNN_FLAG_F32_PARAMS) != 0;
  if (master && !h16) {
    set_error("B200RNN_FLAG_F32_PARAMS needs B200RNN_FLAG_F16 or B200RNN_FLAG_BF16 (the dtype of the other tensors)");
    return B200RNN_ERR_INVALID;
  }
  if (h16 && P > 0) {
    set_error("proj_size is float32 only (B200RNN_FLAG_F16 / _BF16 with B200RNN_FLAG_PROJ)");
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (!(d->dropout_p >= 0.f && d->dropout_p <= 1.f)) {
    set_error("dropout_p must be in [0,1] (got %f)", (double)d->dropout_p);
    return B200RNN_ERR_INVALID;
  }
  const int M = desc_models(d);
  if (M < 1) {
    set_error("models must be >= 1 (got %d)", M);
    return B200RNN_ERR_INVALID;
  }
  if (M > 1 && !d->model_strides) {
    set_error("models %d without model_strides", M);
    return B200RNN_ERR_INVALID;
  }
  if (M > 1 && (P > 0 || h16 || master ||
                (d->flags & (B200RNN_FLAG_FUSED_LN | B200RNN_FLAG_ACCUMULATE_GRADS)))) {
    set_error("models %d: several models in one call are float32 only, without proj_size, the fused LayerNorm or "
              "B200RNN_FLAG_ACCUMULATE_GRADS", M);
    return B200RNN_ERR_UNSUPPORTED;
  }
  o->mode = d->mode;
  o->B = d->batch;
  o->T = d->seq_len;
  o->I = d->input_size;
  o->H = d->hidden_size;
  o->L = d->num_layers;
  o->D = d->num_dirs;
  o->G = gates_of(d->mode);
  o->P = P;
  o->HO = P > 0 ? P : d->hidden_size;
  o->NPAR = P > 0 ? 5 : 4;
  o->TB = (size_t)d->seq_len * d->batch;
  o->GH = (size_t)o->G * o->H;
  o->DH = (size_t)o->D * o->HO;
  o->training = d->training != 0;
  o->p = d->dropout_p;
  o->dt = h16 == B200RNN_FLAG_F16 ? DT_F16 : h16 == B200RNN_FLAG_BF16 ? DT_BF16 : DT_F32;
  o->master = master;
  o->M = M;
  o->ms = M > 1 ? d->model_strides : nullptr;
  return B200RNN_OK;
}

constexpr size_t ALIGN_F = 64;  // floats (256 B)

// ---- reserve layout (floats) ------------------------------------------------------------------
struct ReserveLayout {
  size_t gates[8][2], extra[8][2];  // up to 8 layers; Elman: gates holds h_t, no extra block
  size_t m[8][2];                   // proj_size > 0: o * tanh(c) of every step, [T,B,H] (operand of dW_hr)
  size_t ylayer[8], ydrop[8];
  size_t xln;  // LayerNorm(x) of the folded prologue, kept for the layer-0 wgrad (B200RNN_FLAG_FUSED_LN)
  // 16-bit calls, behind the fp32 layout: the input of layer l + 1 as its GEMM read it (rounded, dropped, rounded
  // again; widened), and the top layer's fp32 output (the BPTT's h_{t-1}; the caller's y is rounded)
  size_t xin[8], ytop;
  size_t total;
};

int make_reserve(const Dims& d, ReserveLayout* r, bool fused_ln = false) {
  if (d.L > 8) {
    set_error("num_layers %d > 8 unsupported", d.L);
    return B200RNN_ERR_UNSUPPORTED;
  }
  size_t off = ALIGN_F;  // [0, ALIGN_F): header {dropout seed, dropout offset} written by the forward
  for (int l = 0; l < d.L; ++l)
    for (int k = 0; k < d.D; ++k) {
      r->gates[l][k] = off;
      off += align_up(d.TB * d.GH, ALIGN_F);
      r->extra[l][k] = off;
      if (!is_elman(d.mode)) off += align_up(d.TB * d.H, ALIGN_F);
      r->m[l][k] = off;
      if (d.P > 0) off += align_up(d.TB * d.H, ALIGN_F);
    }
  for (int l = 0; l + 1 < d.L; ++l) {
    r->ylayer[l] = off;
    off += align_up(d.TB * d.DH, ALIGN_F);
    r->ydrop[l] = off;
    if (d.p > 0.f) off += align_up(d.TB * d.DH, ALIGN_F);
  }
  r->xln = off;
  if (fused_ln) off += align_up(d.TB * (size_t)d.I, ALIGN_F);
  for (int l = 0; l + 1 < d.L; ++l) {
    r->xin[l] = off;
    if (d.dt) off += align_up(d.TB * d.DH, ALIGN_F);
  }
  r->ytop = off;
  if (d.dt) off += align_up(d.TB * d.DH, ALIGN_F);
  r->total = off;
  return B200RNN_OK;
}

// ---- scratch layout (floats) ------------------------------------------------------------------
struct ScratchLayout {
  // forward
  size_t f_gates[2], f_y[2], f_tc;
  size_t f_tc_bytes;
  size_t f_ready;  // int per TC_TILE_M-row tile of the input projection: its finished column tiles (streamed GEMM)
  size_t f_total;
  // backward
  size_t b_dgates[2], b_dghn[2], b_wt[2], b_bpart[2], b_dy, b_gemm;
  size_t b_gemm_bytes;
  // tensor-core backward GEMMs: dense TF32 hi/lo splits of the operands (hi at the offset, lo right behind it)
  size_t b_tc_dg, b_tc_hn, b_tc_x, b_tc_y, b_tc_w, b_tc_part;
  size_t b_tc_part_bytes;
  size_t b_dxln, b_lnpart;  // fused LayerNorm backward: dense d/dLN(x) [TB][I], per-CTA column partials
  size_t b_h0;              // [B][G*H]: gate gradients of each row's first step, paired with h_0 in dW_hh
  size_t b_dhp[2];          // proj_size > 0, per direction [T,B,P]: gradient w.r.t. the projected h_t (dW_hr)
  size_t b_total;
  // both passes, past both layouts: int [B], the batch-slot order of a ragged batch (launch_length_order); the forward
  // and the backward each compute it from `lengths`
  size_t order;
};

// ---- 16-bit calls: fp32 copies behind the scratch layout (floats, from `base`) ---------------------------------------
// forward: the widened biases of every (layer, direction) and the W_hh of one layer's directions (fixed configs), the
//          widened h_0 / c_0, the fp32 h_n / c_n, the 16-bit input of the next layer (a16), and without a reserve the
//          rounded inputs and the top layer's fp32 output
// backward: x, dy, the states and their gradients, every parameter and gradient, dx, all fp32
// fp32 master parameters (B200RNN_FLAG_F32_PARAMS), behind the rest: the 16-bit images of every weight_ih and weight_hh,
//          which the 16-bit kernels read in place of the caller's 16-bit parameters
struct H16Scratch {
  size_t bias[8][2], whh, h0, c0, hn, cn, a16, xin, ytop;
  size_t x32, dy32, dhn, dcn, bh0, bc0, dh0, dc0, w32[8][2], dw32[8][2], dx32;
  size_t ih16[8][2], hh16[8][2];
  size_t total;
};

void make_h16_scratch(const Dims& d, size_t base, H16Scratch* h) {
  size_t off = base;
  auto take = [&](size_t n) { const size_t at = off; off += align_up(n, ALIGN_F); return at; };
  const size_t st = (size_t)d.L * d.D * d.B * d.H;
  for (int l = 0; l < d.L && l < 8; ++l)
    for (int k = 0; k < d.D; ++k) h->bias[l][k] = take(2 * d.GH);
  h->whh = take((size_t)d.D * d.GH * d.H);
  h->h0 = take(st); h->c0 = take(st); h->hn = take(st); h->cn = take(st);
  h->a16 = take((d.TB * (d.I > (int)d.DH ? (size_t)d.I : d.DH) + 1) / 2);
  h->xin = take(d.TB * d.DH);
  h->ytop = take(d.TB * d.DH);
  h->x32 = take(d.TB * d.I); h->dy32 = take(d.TB * d.DH);
  h->dhn = take(st); h->dcn = take(st); h->bh0 = take(st); h->bc0 = take(st); h->dh0 = take(st); h->dc0 = take(st);
  for (int l = 0; l < d.L && l < 8; ++l)
    for (int k = 0; k < d.D; ++k) {
      const size_t n = d.GH * (l == 0 ? (size_t)d.I : d.DH) + d.GH * d.H + 2 * d.GH;
      h->w32[l][k] = take(n);
      h->dw32[l][k] = take(n);
    }
  h->dx32 = take(d.TB * d.I);
  for (int l = 0; l < d.L && l < 8; ++l)
    for (int k = 0; k < d.D; ++k) {
      const size_t Il = l == 0 ? (size_t)d.I : d.DH;
      h->ih16[l][k] = take(d.master ? (d.GH * Il + 1) / 2 : 0);
      h->hh16[l][k] = take(d.master ? (d.GH * d.H + 1) / 2 : 0);
    }
  h->total = off;
}

// split-K partials of the tensor-core gradient GEMMs: <= (#SMs / tiles) * M * N floats
constexpr size_t TC_PART_BYTES = (size_t)160 * 128 * 128 * sizeof(float);

void make_scratch(const Dims& d, ScratchLayout* s) {
  size_t off = ALIGN_F;  // header (dropout seed/offset when nothing is saved for backward)
  for (int k = 0; k < d.D; ++k) {
    s->f_gates[k] = off;
    off += align_up(d.TB * d.GH, ALIGN_F);
  }
  for (int k = 0; k < 2; ++k) {
    s->f_y[k] = off;
    off += align_up(d.TB * d.DH, ALIGN_F);
  }
  // split operands (hi/lo) of the tensor-core 3xTF32 input projection
  {
    const int Kmax = d.I > (int)d.DH ? d.I : (int)d.DH;
    s->f_tc = off;
    s->f_tc_bytes = gemm_tc_scratch_bytes((int)d.TB, (int)d.GH, Kmax);
    off += align_up(s->f_tc_bytes / sizeof(float) + 1, ALIGN_F);
  }
  s->f_ready = off;
  off += align_up((d.TB + TC_TILE_M - 1) / TC_TILE_M, ALIGN_F);
  s->f_total = off;

  off = 0;
  for (int k = 0; k < d.D; ++k) {
    s->b_dgates[k] = off;
    off += align_up(d.TB * d.GH, ALIGN_F);
    s->b_dghn[k] = off;
    off += align_up(d.TB * d.H, ALIGN_F);
    s->b_wt[k] = off;
    off += align_up(d.GH * d.H, ALIGN_F);
    s->b_bpart[k] = off;
    off += align_up((size_t)rec_bwd_max_slices(d.B) * (d.G + 1) * d.H, ALIGN_F);
  }
  s->b_dy = off;
  off += align_up(d.TB * d.DH, ALIGN_F);
  size_t gb = 0;
  const int K = (int)d.TB;
  size_t g0 = gemm_scratch_bytes((int)d.GH, d.I, K);
  size_t g1 = gemm_scratch_bytes((int)d.GH, (int)d.DH, K);
  size_t g2 = gemm_scratch_bytes((int)d.GH, d.H, K);
  gb = g0 > g1 ? g0 : g1;
  gb = gb > g2 ? gb : g2;
  if (d.P > 0) {  // dW_hr [P, H]
    const size_t g3 = gemm_scratch_bytes(d.P, d.H, K);
    gb = gb > g3 ? gb : g3;
  }
  s->b_gemm = off;
  s->b_gemm_bytes = gb;
  off += align_up(gb / sizeof(float) + 1, ALIGN_F);
  {
    const size_t Imax = d.I > (int)d.DH ? (size_t)d.I : d.DH;
    s->b_tc_dg = off;  off += align_up(2 * d.TB * d.GH, ALIGN_F);
    s->b_tc_hn = off;  off += align_up(2 * d.TB * d.H, ALIGN_F);
    s->b_tc_x = off;   off += align_up(2 * d.TB * Imax, ALIGN_F);
    s->b_tc_y = off;   off += align_up(2 * d.TB * d.H, ALIGN_F);
    s->b_tc_w = off;   off += align_up(2 * Imax * d.GH, ALIGN_F);
    s->b_tc_part = off;
    s->b_tc_part_bytes = TC_PART_BYTES;
    off += align_up(s->b_tc_part_bytes / sizeof(float), ALIGN_F);
  }
  s->b_dxln = off;
  off += align_up(d.TB * (size_t)d.I, ALIGN_F);
  s->b_lnpart = off;
  off += align_up(layernorm_bwd_scratch_floats(d.I), ALIGN_F);
  s->b_h0 = off;
  off += align_up((size_t)d.B * d.GH, ALIGN_F);
  for (int k = 0; k < 2; ++k) {
    s->b_dhp[k] = off;
    if (d.P > 0 && k < d.D) off += align_up(d.TB * (size_t)d.P, ALIGN_F);
  }
  s->b_total = off;

  s->order = s->f_total > s->b_total ? s->f_total : s->b_total;
  s->f_total = s->b_total = s->order + align_up((size_t)d.B, ALIGN_F);
}

// One model's reserve and scratch blocks (floats, multiples of ALIGN_F): what b200rnn_workspace_bytes returns for one
// model; model m's blocks start at m times them
void model_blocks(const Dims& d, bool fused_ln, size_t* rs, size_t* ss) {
  ReserveLayout r;
  make_reserve(d, &r, fused_ln);
  ScratchLayout s;
  make_scratch(d, &s);
  size_t stotal = s.f_total > s.b_total ? s.f_total : s.b_total;
  if (d.dt) {
    H16Scratch h;
    make_h16_scratch(d, stotal, &h);
    stotal = h.total;
  }
  *rs = r.total + ALIGN_F;
  *ss = stotal + ALIGN_F;
}

// Model m's parameter table: params[i] offset by m times its model stride (NULL stays NULL)
void model_params(const Dims& d, const float* const* params, int m, const float** out) {
  const int n = d.L * d.D * d.NPAR;
  for (int i = 0; i < n; ++i) out[i] = params[i] ? params[i] + (m ? m * d.ms[2 + i] : 0) : nullptr;
}

// ---- weight cache layout (floats): per (layer, direction) the TF32 hi then lo split of weight_ih [G*H, I_l], then its
// fp16-pair split (gemm_h16_layout.cuh, g16::wcache_layout: the byte offsets, all multiples of 256)
struct WCacheLayout {
  size_t hi[8][2], lo[8][2], h16[8][2];
  bool has_whh16;  // GRU-256, D = 1: per layer weight_hh as the fp16-pair recurrence stages it (h16::Gru256)
  size_t whh16[8];
  size_t total;
};

void make_wcache(const Dims& d, WCacheLayout* w) {
  const g16::WCache b = g16::wcache_layout(d.L, d.D, d.I, (int)d.DH, (int)d.GH);
  for (int l = 0; l < d.L && l < 8; ++l)
    for (int k = 0; k < d.D; ++k) {
      w->hi[l][k] = b.hi[l][k] / sizeof(float);
      w->lo[l][k] = b.lo[l][k] / sizeof(float);
      w->h16[l][k] = b.h16[l][k] / sizeof(float);
    }
  w->has_whh16 = b.has_whh16;
  for (int l = 0; l < d.L && l < 8; ++l) w->whh16[l] = b.whh16[l] / sizeof(float);
  w->total = b.total / sizeof(float);
}

inline bool aligned_to(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }

// ---- gradient GEMMs of the backward pass -----------------------------------------------------------------------
// An fp32 operand [R][C] (row r at p + rows.off(r)) and where the tensor cores take its TF32 split: hi dense [R][C] at
// `split`, lo right behind it (3xTF32 only). The first tensor-core GEMM that reads the operand writes the split.
struct GradSrc {
  const float* p;
  RowMap rows;
  int R, C;
  float* split;
  bool split_done;
};

// One operand of a gradient GEMM, read from row `row0` of its source on. kcontig: the source's rows are the GEMM's m
// (or n) and its columns k; otherwise its rows are k (the operands whose contraction index is the step (t,b)).
struct GradOperand {
  GradSrc* src;
  int row0;
  bool kcontig;
};

// C[M,N] (+)= sum_k A(m,k) B(k,n)
struct GradGemm {
  GradOperand a, b;
  int M, N, K;
  float* C;
  RowMap c_rows;
  int accumulate;
  bool splitk;  // split-K over the long T*B contraction of a wgrad (FFMA: the gemm workspace, tensor cores: b_tc_part)
  bool tc;      // tensor-core presplit GEMM (3xTF32, or single-pass TF32 with `tf32`); FFMA otherwise
  const char* what = "gemm";  // the product, named in the B200RNN_DEBUG line
};

// The K splits a gradient GEMM runs with, as its launcher chooses them: `splitk` splits of `chunk` k-blocks of 32
// (tensor cores) or `chunk` K values (FFMA) each; the last split may be shorter
struct GradPlan {
  int splitk, chunk;
};

GradPlan grad_gemm_plan(const GradGemm& g, const ScratchLayout& sl, float* S) {
  GradPlan p;
  if (g.tc) {
    tc_splitk_plan(g.M, g.N, g.K, g.splitk, g.splitk ? sl.b_tc_part_bytes : 0, &p.splitk, &p.chunk);
  } else {
    const bool ws = g.splitk && sl.b_gemm_bytes;
    gemm_splitk_plan(g.M, g.N, g.K, ws ? S + sl.b_gemm : nullptr, ws ? sl.b_gemm_bytes : 0, &p.splitk, &p.chunk);
  }
  return p;
}

// plan (optional): receives the GradPlan the launch runs with. B200RNN_DEBUG: one line per GEMM (host side only)
int run_grad_gemm(const GradGemm& g, const ScratchLayout& sl, float* S, bool tf32, cudaStream_t st,
                  GradPlan* plan = nullptr) {
  static const bool debug = getenv("B200RNN_DEBUG") != nullptr;
  if (debug || plan) {
    const GradPlan p = grad_gemm_plan(g, sl, S);
    if (plan) *plan = p;
    // the FFMA GEMM is fp32 whatever the TF32 flag says
    if (debug)
      fprintf(stderr,
              "[b200rnn] grad gemm %s: M=%d N=%d K=%d path=%s a=%s b=%s a_row0=%d b_row0=%d splitk=%d %s=%d "
              "accumulate=%d tf32=%d\n",
              g.what, g.M, g.N, g.K, g.tc ? "tc" : "ffma", g.a.kcontig ? "k" : "mn", g.b.kcontig ? "k" : "mn",
              g.a.row0, g.b.row0, p.splitk, g.tc ? "kb_per_split" : "k_chunk", p.chunk, g.accumulate,
              (g.tc && tf32) ? 1 : 0);
  }
  if (!g.tc) {
    GemmParams p;
    memset(&p, 0, sizeof(p));
    p.A = g.a.src->p + g.a.src->rows.off(g.a.row0); p.a_rows = g.a.src->rows; p.a_kcontig = g.a.kcontig;
    p.B = g.b.src->p + g.b.src->rows.off(g.b.row0); p.b_rows = g.b.src->rows; p.b_kcontig = g.b.kcontig;
    p.C = g.C; p.c_rows = g.c_rows;
    p.M = g.M; p.N = g.N; p.K = g.K;
    p.accumulate = g.accumulate;
    const bool ws = g.splitk && sl.b_gemm_bytes;
    return launch_gemm(p, ws ? S + sl.b_gemm : nullptr, ws ? sl.b_gemm_bytes : 0, st);
  }
  TcOperand op[2];
  for (int i = 0; i < 2; ++i) {
    const GradOperand& o = i ? g.b : g.a;
    GradSrc* s = o.src;
    const size_t n = (size_t)s->R * s->C, at = (size_t)o.row0 * s->C;
    if (!s->split_done) {
      const int rc = tc_split(s->p, s->rows, s->R, s->C, s->split, tf32 ? nullptr : s->split + n, st);
      if (rc) return rc;
      s->split_done = true;
    }
    op[i] = TcOperand{s->split + at, tf32 ? nullptr : s->split + n + at, (long long)s->C, !o.kcontig};
  }
  return tc_gemm_presplit(op[0], op[1], g.M, g.N, g.K, g.C, g.c_rows, nullptr, nullptr, 0, g.accumulate,
                          g.splitk ? S + sl.b_tc_part : nullptr, g.splitk ? sl.b_tc_part_bytes : 0, st, nullptr, 0,
                          tf32);
}

// ---- one-step cells ---------------------------------------------------------------------------------------------
struct CellDims {
  int mode, B, I, H, G;
  size_t GH;
  bool save, tf32, accumulate, bias;
  // shapes whose gradient GEMMs may take the tensor cores (N % 128 == 0, every source row a multiple of 4 floats):
  // dx / dW_ih (N = I) and dh / dW_hh (N = H)
  bool tc_x, tc_h;
};

constexpr int CELL_MAX_BATCH = 1 << 20;

int check_cell_desc(const b200rnn_cell_desc* d, CellDims* o) {
  if (!d) {
    set_error("cell: null descriptor");
    return B200RNN_ERR_INVALID;
  }
  if (d->mode != B200RNN_GRU && d->mode != B200RNN_LSTM && !is_elman(d->mode)) {
    set_error("cell: mode must be B200RNN_GRU, B200RNN_LSTM, B200RNN_RNN_TANH or B200RNN_RNN_RELU (got %d)", d->mode);
    return B200RNN_ERR_INVALID;
  }
  constexpr uint32_t known =
      B200RNN_FLAG_SAVE_FOR_BACKWARD | B200RNN_FLAG_TF32 | B200RNN_FLAG_ACCUMULATE_GRADS | B200RNN_FLAG_NO_BIAS;
  if (d->flags & ~known) {
    set_error("cell: unknown flags 0x%x (a cell takes SAVE_FOR_BACKWARD, TF32, ACCUMULATE_GRADS and NO_BIAS)",
              d->flags & ~known);
    return B200RNN_ERR_INVALID;
  }
  if (d->batch < 0 || d->input_size < 1 || d->hidden_size < 1) {
    set_error("cell: bad shape: B=%d I=%d H=%d (B >= 0, I >= 1, H >= 1)", d->batch, d->input_size, d->hidden_size);
    return B200RNN_ERR_INVALID;
  }
  const size_t G = gates_of(d->mode), GH = G * d->hidden_size;
  const size_t K = (size_t)(d->input_size > d->hidden_size ? d->input_size : d->hidden_size);
  if (d->batch > CELL_MAX_BATCH || GH * K > 0x7fffffffu || GH * d->batch > 0x7fffffffu ||
      K * d->batch > 0x7fffffffu) {
    set_error("cell: shape too large: B=%d I=%d H=%d (B <= %d, every operand below 2^31 elements)", d->batch,
              d->input_size, d->hidden_size, CELL_MAX_BATCH);
    return B200RNN_ERR_UNSUPPORTED;
  }
  o->mode = d->mode;
  o->B = d->batch;
  o->I = d->input_size;
  o->H = d->hidden_size;
  o->G = (int)G;
  o->GH = GH;
  o->save = (d->flags & B200RNN_FLAG_SAVE_FOR_BACKWARD) != 0;
  o->tf32 = (d->flags & B200RNN_FLAG_TF32) != 0;
  o->accumulate = (d->flags & B200RNN_FLAG_ACCUMULATE_GRADS) != 0;
  o->bias = (d->flags & B200RNN_FLAG_NO_BIAS) == 0;
  o->tc_x = o->I % 128 == 0 && GH % 4 == 0;
  o->tc_h = o->H % 128 == 0;
  return B200RNN_OK;
}

// saved state (floats): the activated gates [B][G*H] (Elman: h'), then GRU W_hn h + b_hn / LSTM c' [B][H] (Elman:
// none), as the sequence path's reserve holds one step
struct CellSaved {
  size_t gates, extra, total;
};

void make_cell_saved(const CellDims& d, CellSaved* s) {
  s->gates = 0;
  s->extra = align_up((size_t)d.B * d.GH, ALIGN_F);
  s->total = s->extra + (is_elman(d.mode) ? 0 : align_up((size_t)d.B * d.H, ALIGN_F));
}

// backward scratch (floats): gate gradients, bias partial sums, and the gradient GEMMs' workspaces laid out as the
// sequence backward's (split-K partials; a TF32 hi/lo split region per tensor-core source)
struct CellScratch {
  size_t dgx, dgh, part;
  size_t tc_dgx, tc_dgh, tc_x, tc_h, tc_wih, tc_whh;
  ScratchLayout gemm;  // only b_gemm, b_gemm_bytes, b_tc_part, b_tc_part_bytes are used
  size_t total;
};

void make_cell_scratch(const CellDims& d, CellScratch* s) {
  const size_t B = d.B;
  size_t off = 0;
  s->dgx = off;  off += align_up(B * d.GH, ALIGN_F);
  s->dgh = off;  if (d.mode == B200RNN_GRU) off += align_up(B * d.GH, ALIGN_F);
  s->part = off; off += align_up((size_t)cell_bwd_slices(d.B) * (d.G + 1) * d.H, ALIGN_F);
  memset(&s->gemm, 0, sizeof(s->gemm));
  const size_t g0 = gemm_scratch_bytes((int)d.GH, d.I, d.B), g1 = gemm_scratch_bytes((int)d.GH, d.H, d.B);
  s->gemm.b_gemm = off;
  s->gemm.b_gemm_bytes = g0 > g1 ? g0 : g1;
  off += align_up(s->gemm.b_gemm_bytes / sizeof(float) + 1, ALIGN_F);
  s->tc_dgx = off;  if (d.tc_x || d.tc_h) off += align_up(2 * B * d.GH, ALIGN_F);
  s->tc_dgh = off;  if (d.tc_h && d.mode == B200RNN_GRU) off += align_up(2 * B * d.GH, ALIGN_F);
  s->tc_x = off;    if (d.tc_x) off += align_up(2 * B * d.I, ALIGN_F);
  s->tc_wih = off;  if (d.tc_x) off += align_up(2 * d.GH * d.I, ALIGN_F);
  s->tc_h = off;    if (d.tc_h) off += align_up(2 * B * d.H, ALIGN_F);
  s->tc_whh = off;  if (d.tc_h) off += align_up(2 * d.GH * d.H, ALIGN_F);
  s->gemm.b_tc_part = off;
  s->gemm.b_tc_part_bytes = (d.tc_x || d.tc_h) ? TC_PART_BYTES : 0;
  off += align_up(s->gemm.b_tc_part_bytes / sizeof(float), ALIGN_F);
  s->total = off;
}

}  // namespace
}  // namespace b200rnn

using namespace b200rnn;

extern "C" {

B200RNN_API int b200rnn_version(void) { return B200RNN_ABI_VERSION; }

B200RNN_API const char* b200rnn_last_error(void) { return g_err; }

B200RNN_API unsigned long long b200rnn_launch_count(void) { return g_launches.load(); }

/* debug only (not declared in the public header): device buffer of [T][8] int64 phase timestamps */
B200RNN_API void b200rnn_debug_set_trace(long long* dev_buf) { g_trace = dev_buf; }

B200RNN_API int b200rnn_sm_count(void) {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
    set_error("cannot query the CUDA device: %s", cudaGetErrorString(cudaGetLastError()));
    return B200RNN_ERR_CUDA;
  }
  return n;
}

B200RNN_API int b200rnn_workspace_bytes(const b200rnn_desc* desc, size_t* reserve_bytes, size_t* scratch_bytes) {
  Dims d;
  int rc = check_desc(desc, &d);
  if (rc) return rc;
  ReserveLayout r;
  rc = make_reserve(d, &r, (desc->flags & B200RNN_FLAG_FUSED_LN) != 0);
  if (rc) return rc;
  size_t rs, ss;
  model_blocks(d, (desc->flags & B200RNN_FLAG_FUSED_LN) != 0, &rs, &ss);
  if (reserve_bytes) *reserve_bytes = (size_t)d.M * rs * sizeof(float);
  if (scratch_bytes) *scratch_bytes = (size_t)d.M * ss * sizeof(float);
  return B200RNN_OK;
}

// B200RNN_FLAG_F32_PARAMS: one round16_multi launch over the call's L * D * 4 fp32 parameters. Every parameter is
// rounded to the 16-bit dtype once; what the 16-bit call reads from the caller's 16-bit parameters is written from it:
//   forward:  the 16-bit images of weight_ih (hs.ih16) and weight_hh (hs.hh16), the fp32 biases (hs.bias) and, for the
//             fixed configs (whh32), the fp32 weight_hh at its place in hs.w32;
//   backward: every parameter in fp32 (hs.w32, the fp32 BPTT's operands) and the 16-bit weight_hh images.
// img: the parameter table of the rest of the call (images of the weights; biases and fp32 weight_hh read elsewhere)
static int round_master_params(const Dims& d, const float* const* params, float* S, const H16Scratch& hs, bool bwd,
                               bool whh32, const float** img, cudaStream_t st) {
  if (!params) {
    set_error("null parameter table");
    return B200RNN_ERR_INVALID;
  }
  Round16Seg seg[ROUND16_MAX_SEGS];
  int n = 0;
  for (int l = 0; l < d.L; ++l)
    for (int k = 0; k < d.D; ++k) {
      const size_t j = (size_t)(l * d.D + k) * 4;
      const size_t Il = l == 0 ? (size_t)d.I : d.DH;
      for (int i = 0; i < 4; ++i)
        if (!params[j + i]) {
          set_error("null parameter pointer (layer %d dir %d)", l, k);
          return B200RNN_ERR_INVALID;
        }
      uint16_t* ih16 = reinterpret_cast<uint16_t*>(S + hs.ih16[l][k]);
      uint16_t* hh16 = reinterpret_cast<uint16_t*>(S + hs.hh16[l][k]);
      float* w32 = S + hs.w32[l][k];
      const long long nih = (long long)(d.GH * Il), nhh = (long long)(d.GH * d.H), nb = (long long)d.GH;
      float* b32 = bwd ? w32 + nih + nhh : S + hs.bias[l][k];
      seg[n++] = Round16Seg{params[j], bwd ? nullptr : ih16, bwd ? w32 : nullptr, nih};
      // the fixed configs' forward reads weight_hh in fp32 only, everything else the 16-bit image
      const bool hh32 = bwd || whh32;
      seg[n++] = Round16Seg{params[j + 1], (bwd || !whh32) ? hh16 : nullptr, hh32 ? w32 + nih : nullptr, nhh};
      seg[n++] = Round16Seg{params[j + 2], nullptr, b32, nb};
      seg[n++] = Round16Seg{params[j + 3], nullptr, b32 + nb, nb};
      img[j] = reinterpret_cast<const float*>(ih16);
      img[j + 1] = reinterpret_cast<const float*>(hh16);
      img[j + 2] = params[j + 2];
      img[j + 3] = params[j + 3];
    }
  return launch_round16_multi(seg, n, d.dt, ROUND16_IMAGES, st);
}

// The forward of every entry point; h_0 / c_0 NULL = zeros (b200rnn_forward_hx checked their consistency). `shell`:
// called by b200rnn_forward_fused, the model-shell entry, which never takes an initial state; its no-grad forward runs
// the GRU-256 tensor-core recurrence on fp16 pairs (RecFwdParams::shell_nograd)
static int forward_impl(const b200rnn_desc* desc, const float* x, int64_t xs_t, int64_t xs_b,
                        const float* const* params, float* y, int64_t ys_t, int64_t ys_b, float* h_n, float* c_n,
                        void* reserve, void* scratch, uint64_t seed, uint64_t offset, uint64_t* rng_state,
                        const float* ln_gamma, const float* ln_beta, float ln_eps, float* y_pool,
                        const int32_t* lengths, const void* wcache, void* prologue_done, const float* h_0,
                        const float* c_0, bool shell, void* stream_) {
  Dims d;
  int rc = check_desc(desc, &d);
  if (rc) return rc;
  if (shell && (h_0 || c_0)) {
    set_error("forward: the model-shell entry takes no initial state");
    return B200RNN_ERR_INVALID;
  }
  if (d.M > 1 && lengths) {
    set_error("forward: several models in one call take no lengths (ragged batches run one model per call)");
    return B200RNN_ERR_UNSUPPORTED;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  cudaEvent_t prologue_ev = static_cast<cudaEvent_t>(prologue_done);
  if (d.B == 0 || d.T == 0) {
    if (prologue_ev) B200_CUDA_CHECK(cudaEventRecord(prologue_ev, st));
    return B200RNN_OK;
  }
  if (wcache && !aligned_to(wcache, 256)) {
    set_error("forward: the weight cache must be 256-byte aligned");
    return B200RNN_ERR_INVALID;
  }
  WCacheLayout wl;
  make_wcache(d, &wl);
  const float* WC = static_cast<const float*>(wcache);
  const bool save = (desc->flags & B200RNN_FLAG_SAVE_FOR_BACKWARD) != 0;
  if (!x || !params || (!y && !y_pool) || !h_n || (d.mode == B200RNN_LSTM && !c_n)) {
    set_error("forward: null pointer argument");
    return B200RNN_ERR_INVALID;
  }
  if (d.P > 0 && (y_pool || ln_gamma || wcache || prologue_ev || !y)) {
    set_error("forward: the model-shell fusions (LayerNorm prologue, y_pool, weight cache) do not take proj_size");
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (!y && save) {
    set_error("forward: the full output is needed by backward (h_{t-1} of every step): pass y as well as y_pool");
    return B200RNN_ERR_INVALID;
  }
  const bool fused_ln = (desc->flags & B200RNN_FLAG_FUSED_LN) != 0;
  if (fused_ln && !ln_gamma) {
    set_error("forward: B200RNN_FLAG_FUSED_LN without ln_gamma / ln_beta");
    return B200RNN_ERR_INVALID;
  }
  if ((ln_gamma == nullptr) != (ln_beta == nullptr)) {
    set_error("forward: LayerNorm prologue needs both gamma and beta");
    return B200RNN_ERR_INVALID;
  }
  if (save && !reserve) {
    set_error("forward: B200RNN_FLAG_SAVE_FOR_BACKWARD needs a reserve buffer");
    return B200RNN_ERR_INVALID;
  }
  if (!scratch) {
    set_error("forward: a scratch buffer is required");
    return B200RNN_ERR_INVALID;
  }
  if ((reserve && !aligned_to(reserve, 256)) || (scratch && !aligned_to(scratch, 256))) {
    set_error("forward: reserve/scratch must be 256-byte aligned");
    return B200RNN_ERR_INVALID;
  }
  ReserveLayout rl;
  rc = make_reserve(d, &rl, fused_ln);
  if (rc) return rc;
  ScratchLayout sl;
  make_scratch(d, &sl);
  // model m's reserve and scratch blocks start at m * RS and m * SS (one model: R0 and S0 are the whole buffers)
  float* const R0 = static_cast<float*>(reserve);
  float* const S0 = static_cast<float*>(scratch);
  size_t RS, SS;
  model_blocks(d, fused_ln, &RS, &SS);
  float* R = R0;
  float* S = S0;
  const bool drop = d.training && d.p > 0.f && d.L > 1;
  // each model's dropout header {seed, offset} at the start of its block
  auto model_hdr = [&](int m) { return reinterpret_cast<uint64_t*>(save ? R0 + m * RS : S0 + m * SS); };
  uint64_t* hdr = model_hdr(0);
  if (drop || save) {
    // rng_state per model (stride > 0), or one shared state read by every model and advanced by model 0, which comes
    // last: once (stride 0: every model draws the same masks) or M times (stride -1: model m draws what the m-th of M
    // consecutive one-model calls would)
    const int64_t rng_ms = d.M > 1 ? d.ms[1] : 0;
    const uint64_t draw = drop ? (uint64_t)((d.TB * d.DH + 3) / 4) : 0;
    for (int m = d.M - 1; m >= 0; --m) {
      const uint64_t consume = rng_ms > 0 ? draw : m > 0 ? 0 : rng_ms < 0 ? d.M * draw : draw;
      rc = launch_rng_setup(model_hdr(m), seed, offset, rng_state ? rng_state + m * (rng_ms > 0 ? rng_ms : 0) : nullptr,
                            consume, st, rng_ms < 0 ? m * draw : 0);
      if (rc) return rc;
    }
  }
  int* order = nullptr;  // ragged batch: rows sorted into batch slots by length, shared by every layer
  if (lengths) {
    order = reinterpret_cast<int*>(S + sl.order);
    rc = launch_length_order(lengths, d.B, order, st);
    if (rc) return rc;
  }
  // 16-bit call: the fp32 kernels read exact fp32 copies of the biases and states; h_n / c_n (and y) are produced in
  // fp32 and rounded once at the end, the input projection reads the 16-bit operands natively
  const int dt = d.dt;
  H16Scratch hs;
  void* const y16 = y;
  void* const hn16 = h_n;
  void* const cn16 = c_n;
  // fp32 master parameters: one launch rounds them into what the 16-bit call reads (16-bit images of weight_ih and
  // weight_hh, the fp32 biases, the fixed configs' fp32 weight_hh), and the rest of the call runs on the images
  const float* img[8 * 2 * 4];
  const bool fixed_whh = !is_elman(d.mode) && (d.H == 128 || d.H == 256);
  if (dt) {
    make_h16_scratch(d, sl.b_total, &hs);
    if (d.master) {
      rc = round_master_params(d, params, S, hs, false, fixed_whh, img, st);
      if (rc) return rc;
      params = img;
    }
    for (int l = 0; l < d.L && !d.master; ++l)
      for (int k = 0; k < d.D; ++k) {
        const float* const* pp = params + (size_t)(l * d.D + k) * d.NPAR;
        if (!pp[2] || !pp[3]) {
          set_error("forward: null parameter pointer (layer %d dir %d)", l, k);
          return B200RNN_ERR_INVALID;
        }
        for (int i = 0; i < 2; ++i) {
          rc = launch_widen16(pp[2 + i], simple_rows(d.GH), 1, (int)d.GH, dt, S + hs.bias[l][k] + i * d.GH, st);
          if (rc) return rc;
        }
      }
    const int nst = d.L * d.D * d.B;
    if (h_0) {
      rc = launch_widen16(h_0, simple_rows(d.H), nst, d.H, dt, S + hs.h0, st);
      if (rc) return rc;
      h_0 = S + hs.h0;
    }
    if (c_0) {
      rc = launch_widen16(c_0, simple_rows(d.H), nst, d.H, dt, S + hs.c0, st);
      if (rc) return rc;
      c_0 = S + hs.c0;
    }
    h_n = S + hs.hn;
    if (c_n) c_n = S + hs.cn;
  }

  const bool tc = tc_available();
  // single-pass TF32 GEMMs and tc8 recurrence; fp32 calls only: 16-bit modules keep their numerics whatever torch's fp32
  // matmul precision says, as cuDNN's 16-bit RNNs do
  const bool tf32 = (desc->flags & B200RNN_FLAG_TF32) != 0 && !dt;
  int sms = NUM_SMS;
  {
    int dev = 0;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  // ready counters of a streamed input projection; a kernel that writes the GEMM's A operand (LayerNorm, dense copy,
  // dropout) zeroes them, so each layer (and each CUDA-graph replay) starts from zero; an A operand read straight from
  // the caller's tensor or the previous layer's output takes a memset
  int* ready = reinterpret_cast<int*>(S + sl.f_ready);
  const int tiles_m = (int)((d.TB + TC_TILE_M - 1) / TC_TILE_M);
  bool ready_zeroed = false;  // this layer's dropout pass zeroed the counters for the next layer
  const float* pm[8 * 2 * 5];  // model m's parameter table
  for (int l = 0; l < d.L; ++l) {
    const int Il = l == 0 ? d.I : (int)d.DH;
    // ---- the recurrence config, chosen before anything of the layer is enqueued
    RecFwdParams rp;
    memset(&rp, 0, sizeof(rp));
    rp.mode = d.mode; rp.B = d.B; rp.T = d.T; rp.H = d.H; rp.D = d.D;
    rp.training = save ? 1 : 0;
    rp.lengths = lengths;
    rp.order = order;
    rp.tf32 = tf32 ? 1 : 0;
    rp.shell_nograd = shell && !save ? 1 : 0;
    rp.P = d.P;
    // frozen GRU-256 weights: the fp16-pair recurrence copies its W_hh pairs from the cache instead of splitting them
    if (WC && wl.has_whh16) rp.whh16[0] = WC + wl.whh16[l];
    RecFwdLaunch rec;
    // 16-bit: the runtime-sized kernels read weight_hh as it lies; the fixed configs get fp32 copies below
    rc = plan_rec_fwd(rp, &rec, dt, d.M);
    if (rc) return rc;
    const bool tc_layer = !dt && tc && (Il % 32 == 0) && (d.GH % 128 == 0);
    // Stream the input projection into the recurrence (DESIGN.md §4): the GEMM runs beside the recurrence and publishes
    // its row tiles in time order, the recurrence starts while it runs and waits per step for the tiles it reads. Only
    // when the recurrence is unidirectional (it walks t upwards), fits one wave of 4-CTA clusters and takes at most half
    // of the SMs; the GEMM runs as 4-CTA clusters in the cluster slots the recurrence leaves free. Otherwise GEMM and
    // recurrence run one after the other.
    const int gemm_clusters = rec.capacity - rec.nclusters;
    // The runtime-sized kernels (rec.anyh) take no streamed x-projection.
    const bool stream_xproj = !rec.anyh && d.D == 1 && d.P == 0 && tc_layer && rec.C == 4 && rec.one_wave() &&
                              2 * rec.ctas() <= sms && gemm_clusters > 0;
    // Several models: each model's layer input and input projection in turn, into its own blocks; the recurrence
    // below runs them all
    for (int m = 0; m < d.M; ++m) {
      R = R0 + m * RS;
      S = S0 + m * SS;
      const float* const xm = m ? x + m * d.ms[0] : x;
      if (m) {
        model_params(d, params, m, pm);
      }
      const float* const* const params_m = m ? pm : params;
      // ---- layer input ---------------------------------------------------------------------------
      const float* in;
      RowMap in_rows;
      if (l == 0) {
        in = xm;
        in_rows = tb_rows(xs_t, xs_b, d.B);
      } else {
        if (save)
          in = R + (drop ? rl.ydrop[l - 1] : rl.ylayer[l - 1]);
        else
          in = S + sl.f_y[(l - 1) & 1];
        in_rows = simple_rows((long long)d.DH);
      }
      // 16-bit: the A operand of the native input projection, read in place when the TMA can (else a dense copy)
      const void* a16 = l == 0 ? static_cast<const void*>(x) : S + hs.a16;
      RowMap a16_rows = l == 0 ? tb_rows(xs_t, xs_b, d.B) : simple_rows((long long)d.DH);
      bool n16 = false;
      const char* a16_route = "tma";  // B200RNN_DEBUG: where the 16-bit A operand comes from
      if (dt) {
        n16 = tc && tc_gemm_n16_ok(a16, a16_rows, params[(size_t)l * d.D * d.NPAR], (int)d.TB, (int)d.GH, Il);
        if (!n16 && l == 0 && tc && tc_gemm_n16_ok(S + hs.a16, simple_rows(Il), params[0], (int)d.TB, (int)d.GH, Il)) {
          rc = launch_copy16(x, a16_rows, (int)d.TB, Il, S + hs.a16, st);
          if (rc) return rc;
          a16 = S + hs.a16;
          a16_rows = simple_rows(Il);
          a16_route = "copy16";
          n16 = true;
        }
      }
      // ---- A operand of the tensor-core input projection (fp32, split on chip by the GEMM), shared by the directions:
      // the layer input itself when the GEMM can read it in place, else a dense copy in the GEMM's workspace
      void* tc_ws = S + sl.f_tc;
      const float* a_in = in;
      RowMap a_rows = in_rows;
      const char* a_route = "tma";  // B200RNN_DEBUG: where the fp32 A operand comes from
      if (tc_layer) {
        float* a_dense = tc_a_hi(tc_ws);
        if (l == 0 && ln_gamma) {
          float* out = (save && fused_ln) ? R + rl.xln : a_dense;
          // padded rows of a ragged batch are written as 0: the backward's dW_ih GEMM reads this saved operand
          rc = tc_layernorm(in, in_rows, (int)d.TB, Il, ln_gamma, ln_beta, ln_eps, out, st, ready, tiles_m, lengths, d.B);
          a_in = out;
          a_rows = simple_rows(Il);
          a_route = "ln";
        } else if (!tc_a_f32_in_place(in, in_rows, (int)d.TB, Il)) {
          rc = tc_gather_rows(in, in_rows, (int)d.TB, Il, a_dense, st, ready, tiles_m);
          a_in = a_dense;
          a_rows = simple_rows(Il);
          a_route = "gather";
        } else if (stream_xproj && !ready_zeroed) {
          B200_CUDA_CHECK(cudaMemsetAsync(ready, 0, tiles_m * sizeof(int), st));
        }
        if (rc) return rc;
      } else if (l == 0 && ln_gamma) {
        set_error("forward: the fused LayerNorm prologue needs the tensor-core input projection (input_size %% 32 == 0)");
        return B200RNN_ERR_UNSUPPORTED;
      }
      // everything before the first GEMM is enqueued: kernels of a stream gated on this event become pending no earlier
      // than the layer-0 GEMM, which then wins the SMs on this stream's priority
      if (l == 0 && prologue_ev) B200_CUDA_CHECK(cudaEventRecord(prologue_ev, st));
      ready_zeroed = false;
      for (int k = 0; k < d.D; ++k) {
        const float* const* pp = params_m + (size_t)(l * d.D + k) * d.NPAR;
        const float *w_ih = pp[0], *w_hh = pp[1], *b_ih = pp[2], *b_hh = pp[3];
        if (!w_ih || !w_hh || !b_ih || !b_hh || (d.P > 0 && !pp[4])) {
          set_error("forward: null parameter pointer (layer %d dir %d)", l, k);
          return B200RNN_ERR_INVALID;
        }
        if (!aligned_to(w_hh, 16)) {
          set_error("forward: weight_hh must be 16-byte aligned for the TMA bulk copy (layer %d dir %d)", l, k);
          return B200RNN_ERR_INVALID;
        }
        float* gates = save ? R + rl.gates[l][k] : S + sl.f_gates[k];
        if (dt) {  // K1 on 16-bit operands: native f16 / bf16 wgmma, else the FFMA GEMM on exact fp32 copies
          const float* b32 = S + hs.bias[l][k];
          const int b2n = d.mode == B200RNN_GRU ? 2 * d.H : (int)d.GH;
          // each direction's weight_ih checked on its own: one the TMA cannot read takes the FFMA GEMM
          if (n16 && tc_gemm_n16_ok(a16, a16_rows, w_ih, (int)d.TB, (int)d.GH, Il)) {
            rc = tc_gemm_n16(a16, a16_rows, w_ih, (int)d.TB, (int)d.GH, Il, dt, gates, simple_rows((long long)d.GH), b32,
                             b32 + d.GH, b2n, st, a16_route);
          } else {
            float* aw = S + sl.f_tc;
            float* ww = aw + align_up(d.TB * Il, ALIGN_F);
            rc = launch_widen16(a16, a16_rows, (int)d.TB, Il, dt, aw, st);
            if (!rc) rc = launch_widen16(w_ih, simple_rows(Il), (int)d.GH, Il, dt, ww, st);
            if (rc) return rc;
            GemmParams g;
            memset(&g, 0, sizeof(g));
            g.A = aw; g.a_rows = simple_rows(Il); g.a_kcontig = 1;
            g.B = ww; g.b_rows = simple_rows(Il); g.b_kcontig = 1;
            g.C = gates; g.c_rows = simple_rows((long long)d.GH);
            g.M = (int)d.TB; g.N = (int)d.GH; g.K = Il;
            g.bias1 = b32; g.bias2 = b32 + d.GH; g.bias2_n = b2n;
            g.a_route = "widen";
            rc = launch_gemm(g, nullptr, 0, st);
          }
          if (rc) return rc;
        } else {
          // K1: x-projection of every time step at once, biases folded (GRU: b_hh only for r,z; LSTM, Elman: all of it)
          GemmParams g;
          memset(&g, 0, sizeof(g));
          g.A = a_in; g.a_rows = a_rows; g.a_kcontig = 1;
          g.B = w_ih; g.b_rows = simple_rows(Il); g.b_kcontig = 1;
          g.C = gates; g.c_rows = simple_rows((long long)d.GH);
          g.M = (int)d.TB; g.N = (int)d.GH; g.K = Il;
          g.bias1 = b_ih; g.bias2 = b_hh;
          g.bias2_n = d.mode == B200RNN_GRU ? 2 * d.H : (int)d.GH;
          g.a_route = a_route;
          if (tc_layer) {
            g.tc_ws = tc_ws;
            g.tc_ws_bytes = sl.f_tc_bytes;
            g.tc_a_f32 = 1;
            g.tc_tf32 = tf32 ? 1 : 0;
            // the no-grad forward of b200rnn_forward_fused in default precision: fp16 pairs (the rule of the fp16-pair
            // recurrence, RecFwdParams::shell_nograd)
            g.tc_h16 = rp.shell_nograd && !tf32 && g16::shape_ok((int)d.GH, Il) ? 1 : 0;
            if (WC) {  // weight_ih was split once by b200rnn_prepare_weights (frozen encoders); TF32 reads only hi
              g.tc_b_hi = WC + wl.hi[l][k];
              g.tc_b_lo = tf32 ? nullptr : WC + wl.lo[l][k];
              if (g.tc_h16) g.tc_b_h16 = WC + wl.h16[l][k];
            }
            if (stream_xproj && gemm_tc_eligible(g, g.tc_ws_bytes)) {
              g.tc_ready = ready;
              g.tc_stream_clusters = gemm_clusters;
              rp.ready = ready;
              rp.tiles_n = (int)d.GH / TC_TILE_N;
            }
          }
          rc = launch_gemm(g, nullptr, 0, st);
          if (rc) return rc;
        }
        if (m > 0) continue;  // the recurrence takes model 0's pointers and the model strides
        rp.w_hh[k] = w_hh;
        rp.b_hh[k] = b_hh;
        if (dt) {
          rp.b_hh[k] = S + hs.bias[l][k] + d.GH;
          if (!rec.anyh && d.master) {  // rounded into hs.w32 by round_master_params
            if (!fixed_whh) {
              set_error("forward: no fp32 weight_hh for the recurrence config (mode %d, hidden_size %d)", d.mode, d.H);
              return B200RNN_ERR_UNSUPPORTED;
            }
            rp.w_hh[k] = S + hs.w32[l][k] + d.GH * (size_t)Il;
          } else if (!rec.anyh) {  // the fixed configs read fp32: an exact copy per direction
            float* w32 = S + hs.whh + (size_t)k * d.GH * d.H;
            rc = launch_widen16(w_hh, simple_rows(d.H), (int)d.GH, d.H, dt, w32, st);
            if (rc) return rc;
            rp.w_hh[k] = w32;
          }
        }
        rp.gates[k] = gates;
        rp.extra[k] = save && !is_elman(d.mode) ? R + rl.extra[l][k] : nullptr;
        if (d.P > 0) {
          rp.w_hr[k] = pp[4];
          rp.m[k] = save ? R + rl.m[l][k] : nullptr;
        }
      }
    }
    R = R0;
    S = S0;
    if (d.M > 1) {
      RecModels& mo = rec.models;
      for (int k = 0; k < d.D; ++k) {
        const int64_t* msp = d.ms + 2 + (size_t)(l * d.D + k) * d.NPAR;
        mo.whh[k] = msp[1];
        mo.bhh[k] = msp[3];
      }
      mo.saved = (long long)(save ? RS : SS);
      mo.y = l == d.L - 1 ? (long long)(d.TB * d.DH) : mo.saved;
      mo.state = (long long)d.L * d.D * d.B * d.H;
    }
    float* ylay = nullptr;
    if (l == d.L - 1 && dt) {  // fp32, kept for the backward; rounded into the caller's y below
      rp.y = save ? R + rl.ytop : S + hs.ytop;
      rp.y_st = (long long)d.B * d.DH; rp.y_sb = (long long)d.DH;
    } else if (l == d.L - 1) {
      rp.y = y; rp.y_st = ys_t; rp.y_sb = ys_b;
      rp.y_pool = y_pool;
    } else {
      ylay = save ? R + rl.ylayer[l] : S + sl.f_y[l & 1];
      rp.y = ylay;
      rp.y_st = (long long)d.B * d.DH; rp.y_sb = (long long)d.DH;
    }
    rp.h_n = h_n + (size_t)l * d.D * d.B * d.HO;
    rp.c_n = c_n ? c_n + (size_t)l * d.D * d.B * d.H : nullptr;
    rp.h_0 = h_0 ? h_0 + (size_t)l * d.D * d.B * d.HO : nullptr;
    rp.c_0 = c_0 ? c_0 + (size_t)l * d.D * d.B * d.H : nullptr;
    rp.trace = g_trace;
    // Streamed, this launch directly follows the GEMM in the stream (nothing may be enqueued between them) and never
    // comes first: launched after the GEMM, the recurrence waits only on a kernel whose CTAs have all started.
    rc = launch_rec_fwd(rec, rp, st);
    if (rc) return rc;
    if (dt) {
      // 16-bit: the output is rounded once; an inner layer's output is rounded before the dropout and again after it,
      // as stock torch materialises it, and becomes the next layer's 16-bit A operand (its fp32 widening is kept for
      // the backward's dW_ih)
      const RowMap dense = simple_rows((long long)d.DH);
      const int TB = (int)d.TB, DH = (int)d.DH;
      if (l + 1 < d.L) {
        float* xin = save ? R + rl.xin[l] : S + hs.xin;
        void* next = S + hs.a16;
        if (drop) {
          rc = launch_narrow16(ylay, dense, TB, DH, dt, next, dense, false, xin, st);
          if (!rc) rc = launch_dropout(xin, xin, d.TB * d.DH, d.p, hdr, (uint32_t)l, st);
          if (!rc) rc = launch_narrow16(xin, dense, TB, DH, dt, next, dense, false, xin, st);
        } else {
          rc = launch_narrow16(ylay, dense, TB, DH, dt, next, dense, false, save ? xin : nullptr, st);
        }
      } else {
        rc = launch_narrow16(rp.y, dense, TB, DH, dt, y16, tb_rows(ys_t, ys_b, d.B), false, nullptr, st);
      }
      if (rc) return rc;
    } else if (drop && l + 1 < d.L) {  // K7; keeps the raw output when it is needed by backward, else in place
      for (int m = 0; m < d.M; ++m) {  // each model with its own header
        const size_t at = m * (save ? RS : SS);
        float* dropped = save ? R + at + rl.ydrop[l] : ylay + at;
        // the next layer's GEMM reads `dropped` in place; the same launch zeroes its ready counters
        rc = launch_dropout(ylay + at, dropped, d.TB * d.DH, d.p, model_hdr(m), (uint32_t)l, st, m ? nullptr : ready,
                            tiles_m);
        if (rc) return rc;
      }
      ready_zeroed = true;
    }
  }
  if (dt) {
    const int nst = d.L * d.D * d.B;
    rc = launch_narrow16(h_n, simple_rows(d.H), nst, d.H, dt, hn16, simple_rows(d.H), false, nullptr, st);
    if (!rc && cn16) rc = launch_narrow16(c_n, simple_rows(d.H), nst, d.H, dt, cn16, simple_rows(d.H), false, nullptr, st);
    if (rc) return rc;
  }
  return B200RNN_OK;
}

// h_0 / c_0 / dh_0 / dc_0 of the hx entry points: c_0 (dc_0) only for the LSTM, and there c_0 only together with h_0
static int check_initial_state(const b200rnn_desc* desc, const float* h_0, const void* c_0, const void* dc_0,
                               const char* what) {
  if (desc && desc->mode != B200RNN_LSTM && (c_0 || dc_0)) {
    set_error("%s: a %s has no cell state (c_0 / dc_0 must be NULL)", what, mode_name(desc->mode));
    return B200RNN_ERR_INVALID;
  }
  if (c_0 && !h_0) {
    set_error("%s: c_0 without h_0 (pass both initial states, or neither)", what);
    return B200RNN_ERR_INVALID;
  }
  return B200RNN_OK;
}

B200RNN_API int b200rnn_forward_fused(const b200rnn_desc* desc, const float* x, int64_t xs_t, int64_t xs_b,
                                      const float* const* params, float* y, int64_t ys_t, int64_t ys_b, float* h_n,
                                      float* c_n, void* reserve, void* scratch, uint64_t seed, uint64_t offset,
                                      uint64_t* rng_state, const float* ln_gamma, const float* ln_beta, float ln_eps,
                                      float* y_pool, const int32_t* lengths, const void* wcache,
                                      void* prologue_done, void* stream_) {
  if (desc && desc_proj(desc) != 0) {
    set_error("forward_fused: the model-shell entry points do not take proj_size (use b200rnn_forward_hx)");
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (check_shell_desc(desc, "forward_fused")) return B200RNN_ERR_UNSUPPORTED;
  return forward_impl(desc, x, xs_t, xs_b, params, y, ys_t, ys_b, h_n, c_n, reserve, scratch, seed, offset, rng_state,
                      ln_gamma, ln_beta, ln_eps, y_pool, lengths, wcache, prologue_done, nullptr, nullptr, true,
                      stream_);
}

B200RNN_API int b200rnn_forward_hx(const b200rnn_desc* desc, const float* x, int64_t xs_t, int64_t xs_b,
                                   const float* const* params, float* y, int64_t ys_t, int64_t ys_b, const float* h_0,
                                   const float* c_0, float* h_n, float* c_n, void* reserve, void* scratch,
                                   uint64_t seed, uint64_t offset, uint64_t* rng_state, const int32_t* lengths,
                                   void* stream_) {
  Dims d;
  int rc = check_desc(desc, &d);
  if (rc) return rc;
  rc = check_initial_state(desc, h_0, c_0, nullptr, "forward_hx");
  if (rc) return rc;
  if (d.B > 0 && d.T == 0 && h_n && h_0) {  // no step: the final state is the initial one
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    const size_t es = d.dt ? 2 : sizeof(float);
    const size_t bytes = (size_t)d.L * d.D * d.B * d.H * es;
    B200_CUDA_CHECK(cudaMemcpyAsync(h_n, h_0, (size_t)d.L * d.D * d.B * d.HO * es, cudaMemcpyDeviceToDevice,
                                    st));
    if (c_n) {
      if (c_0) B200_CUDA_CHECK(cudaMemcpyAsync(c_n, c_0, bytes, cudaMemcpyDeviceToDevice, st));
      else B200_CUDA_CHECK(cudaMemsetAsync(c_n, 0, bytes, st));
    }
    return B200RNN_OK;
  }
  return forward_impl(desc, x, xs_t, xs_b, params, y, ys_t, ys_b, h_n, c_n, reserve, scratch, seed, offset, rng_state,
                      nullptr, nullptr, 0.f, nullptr, lengths, nullptr, nullptr, h_0, c_0, false, stream_);
}

B200RNN_API int b200rnn_forward(const b200rnn_desc* desc, const float* x, int64_t xs_t, int64_t xs_b,
                                const float* const* params, float* y, int64_t ys_t, int64_t ys_b, float* h_n,
                                float* c_n, void* reserve, void* scratch, uint64_t seed, uint64_t offset,
                                uint64_t* rng_state, void* stream_) {
  return forward_impl(desc, x, xs_t, xs_b, params, y, ys_t, ys_b, h_n, c_n, reserve, scratch, seed, offset, rng_state,
                      nullptr, nullptr, 0.f, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, false, stream_);
}

B200RNN_API int b200rnn_wcache_bytes(const b200rnn_desc* desc, size_t* bytes) {
  Dims d;
  int rc = check_desc(desc, &d);
  if (rc) return rc;
  if (d.L > 8) {
    set_error("num_layers %d > 8 unsupported", d.L);
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (d.P > 0) {
    set_error("wcache_bytes: the weight cache of b200rnn_forward_fused does not take proj_size");
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (check_shell_desc(desc, "wcache_bytes")) return B200RNN_ERR_UNSUPPORTED;
  WCacheLayout wl;
  make_wcache(d, &wl);
  if (bytes) *bytes = (wl.total + ALIGN_F) * sizeof(float);
  return B200RNN_OK;
}

B200RNN_API int b200rnn_prepare_weights(const b200rnn_desc* desc, const float* const* params, void* wcache,
                                        void* stream_) {
  Dims d;
  int rc = check_desc(desc, &d);
  if (rc) return rc;
  if (!params || !wcache || !aligned_to(wcache, 256) || d.L > 8) {
    set_error("prepare_weights: null / misaligned argument");
    return B200RNN_ERR_INVALID;
  }
  if (d.P > 0) {
    set_error("prepare_weights: the weight cache of b200rnn_forward_fused does not take proj_size");
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (check_shell_desc(desc, "prepare_weights")) return B200RNN_ERR_UNSUPPORTED;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  WCacheLayout wl;
  make_wcache(d, &wl);
  float* WC = static_cast<float*>(wcache);
  for (int l = 0; l < d.L; ++l) {
    const int Il = l == 0 ? d.I : (int)d.DH;
    for (int k = 0; k < d.D; ++k) {
      const float* w_ih = params[(size_t)(l * d.D + k) * 4];
      if (!w_ih) {
        set_error("prepare_weights: null weight_ih (layer %d dir %d)", l, k);
        return B200RNN_ERR_INVALID;
      }
      if (Il % 4 != 0) continue;  // such a layer takes the FFMA projection, which reads the fp32 weights directly
      rc = tc_split(w_ih, simple_rows(Il), (int)d.GH, Il, WC + wl.hi[l][k], WC + wl.lo[l][k], st);
      if (rc) return rc;
      if (g16::shape_ok((int)d.GH, Il)) {  // the same split the uncached no-grad forward makes per call
        rc = tc_split_w16(w_ih, simple_rows(Il), (int)d.GH, Il, WC + wl.h16[l][k], st);
        if (rc) return rc;
      }
    }
    if (wl.has_whh16) {  // weight_hh: the pairs the fp16-pair recurrence's prologue makes per launch when uncached
      const float* w_hh = params[(size_t)l * d.D * 4 + 1];
      if (!w_hh || !aligned_to(w_hh, 16)) {
        set_error("prepare_weights: null or misaligned weight_hh (layer %d)", l);
        return B200RNN_ERR_INVALID;
      }
      rc = prep_whh_h16(w_hh, WC + wl.whh16[l], st);
      if (rc) return rc;
    }
  }
  return B200RNN_OK;
}

// The backward of every entry point; h_0 / c_0 NULL = zeros, dh_0 / dc_0 NULL = not computed
static int backward_impl(const b200rnn_desc* desc, const float* x, int64_t xs_t, int64_t xs_b,
                         const float* const* params, const float* y, int64_t ys_t, int64_t ys_b, const float* dy,
                         int64_t dys_t, int64_t dys_b, const float* dy_pool, float dy_pool_scale, const float* dh_n,
                         const float* dc_n, const void* reserve, void* scratch, float* dx, int64_t dxs_t,
                         int64_t dxs_b, float* const* dparams, const int32_t* lengths, const float* ln_gamma,
                         float ln_eps, float* dln_gamma, float* dln_beta, const float* h_0, const float* c_0,
                         float* dh_0, float* dc_0, void* stream_, const float* const* layer_in = nullptr,
                         int w16 = 0, const void* const* whh16 = nullptr) {
  Dims d;
  int rc = check_desc(desc, &d);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (d.B == 0 || d.T == 0) return B200RNN_OK;
  if (!x || !params || !y || (!dy && !dy_pool) || !reserve || !scratch || !dparams) {
    set_error("backward: null pointer argument");
    return B200RNN_ERR_INVALID;
  }
  const bool fused_ln = (desc->flags & B200RNN_FLAG_FUSED_LN) != 0;
  if (fused_ln != (ln_gamma != nullptr)) {
    set_error("backward: B200RNN_FLAG_FUSED_LN and ln_gamma must be given together (as in the forward)");
    return B200RNN_ERR_INVALID;
  }
  if (d.P > 0 && (fused_ln || dy_pool || !dy)) {
    set_error("backward: the model-shell fusions (LayerNorm, pooled gradient) do not take proj_size");
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (fused_ln && (!(d.I == 128 || d.I == 256 || d.I == 512 || d.I == 1024) || !tc_available())) {
    set_error("backward: the fused LayerNorm needs input_size 128, 256, 512 or 1024");
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (!aligned_to(reserve, 256) || !aligned_to(scratch, 256)) {
    set_error("backward: reserve/scratch must be 256-byte aligned");
    return B200RNN_ERR_INVALID;
  }
  ReserveLayout rl;
  rc = make_reserve(d, &rl, fused_ln);
  if (rc) return rc;
  ScratchLayout sl;
  make_scratch(d, &sl);
  if (d.M > 1 && lengths) {
    set_error("backward: several models in one call take no lengths (ragged batches run one model per call)");
    return B200RNN_ERR_UNSUPPORTED;
  }
  // model m's reserve and scratch blocks start at m * RS and m * SS (one model: R0 and S0 are the whole buffers)
  const float* const R0 = static_cast<const float*>(reserve);
  float* const S0 = static_cast<float*>(scratch);
  size_t RS, SS;
  model_blocks(d, fused_ln, &RS, &SS);
  const float* R = R0;
  float* S = S0;
  const bool drop = d.training && d.p > 0.f && d.L > 1;
  const int accumulate = (desc->flags & B200RNN_FLAG_ACCUMULATE_GRADS) ? 1 : 0;
  const bool tf32 = (desc->flags & B200RNN_FLAG_TF32) != 0;  // single-pass TF32 tensor-core GEMMs: hi operands only
  const int TB = (int)d.TB, GH = (int)d.GH;
  int* order = nullptr;  // the forward's slot order, recomputed from the same lengths (nothing of it is in the reserve)
  if (lengths) {
    order = reinterpret_cast<int*>(S + sl.order);
    rc = launch_length_order(lengths, d.B, order, st);
    if (rc) return rc;
  }

  const float* pm[8 * 2 * 5];  // model m's parameter table
  float* dpm[8 * 2 * 5];       // ... and gradient targets
  for (int l = d.L - 1; l >= 0; --l) {
    const int Il = l == 0 ? d.I : (int)d.DH;
    RecBwdParams bp;
    memset(&bp, 0, sizeof(bp));
    bp.mode = d.mode; bp.B = d.B; bp.T = d.T; bp.H = d.H; bp.D = d.D;
    bp.P = d.P;
    if (l == d.L - 1) {
      bp.y = y; bp.y_st = ys_t; bp.y_sb = ys_b;
      bp.dy = dy; bp.dy_st = dys_t; bp.dy_sb = dys_b;
      bp.dy_pool = dy_pool; bp.dy_scale = dy_pool_scale;
    } else {
      bp.y = R + rl.ylayer[l]; bp.y_st = (long long)d.B * d.DH; bp.y_sb = (long long)d.DH;
      bp.dy = S + sl.b_dy; bp.dy_st = (long long)d.B * d.DH; bp.dy_sb = (long long)d.DH;
    }
    const size_t lstate = (size_t)l * d.D * d.B * d.H;    // this layer's [D,B,H] slice of the [L*D,B,H] cell states
    const size_t lhstate = (size_t)l * d.D * d.B * d.HO;  // ... and of the [L*D,B,HO] hidden states
    bp.dh_n = dh_n ? dh_n + lhstate : nullptr;
    bp.dc_n = dc_n ? dc_n + lstate : nullptr;
    bp.h_0 = h_0 ? h_0 + lhstate : nullptr;
    bp.c_0 = c_0 ? c_0 + lstate : nullptr;
    bp.dh_0 = dh_0 ? dh_0 + lhstate : nullptr;
    bp.dc_0 = dc_0 ? dc_0 + lstate : nullptr;
    for (int k = 0; k < d.D; ++k) {
      const float* const* pp = params + (size_t)(l * d.D + k) * d.NPAR;
      if (!pp[0] || !pp[1] || (d.P > 0 && !pp[4])) {
        set_error("backward: null parameter pointer (layer %d dir %d)", l, k);
        return B200RNN_ERR_INVALID;
      }
      bp.w_hh[k] = pp[1];
      bp.w_prep[k] = S + sl.b_wt[k];
      bp.gates[k] = R + rl.gates[l][k];
      bp.extra[k] = is_elman(d.mode) ? nullptr : R + rl.extra[l][k];
      bp.dgates[k] = S + sl.b_dgates[k];
      bp.dghn[k] = S + sl.b_dghn[k];
      bp.dbias_part[k] = S + sl.b_bpart[k];
      if (d.P > 0) {
        bp.w_hr[k] = pp[4];
        bp.dhp[k] = S + sl.b_dhp[k];
      }
    }
    bp.lengths = lengths;
    bp.order = order;
    RecModels mo;  // the caller's tensors are dense per model but for x and the parameters (desc->model_strides)
    if (d.M > 1) {
      mo.M = d.M;
      for (int k = 0; k < d.D; ++k) {
        mo.whh[k] = d.ms[2 + (size_t)(l * d.D + k) * d.NPAR + 1];
        mo.wprep[k] = mo.whh[k] ? (long long)SS : 0;  // a shared weight_hh is transposed once, into model 0's scratch
      }
      mo.saved = (long long)RS;
      mo.y = l == d.L - 1 ? (long long)(d.TB * d.DH) : (long long)RS;
      mo.dy = l == d.L - 1 ? (long long)(d.TB * d.DH) : (long long)SS;
      mo.scr = (long long)SS;
      mo.state = (long long)d.L * d.D * d.B * d.H;
    }
    // 16-bit: whh16 holds each (layer, direction)'s weight_hh as the caller passed it, staged in 16 bits by the
    // runtime-sized BPTT
    rc = launch_rec_bwd(bp, st, w16, whh16 ? whh16 + (size_t)l * d.D : nullptr, d.M > 1 ? &mo : nullptr);
    if (rc) return rc;

    // Several models: the gradient GEMMs of each model in turn, on its own blocks
    for (int m = 0; m < d.M; ++m) {
      R = R0 + m * RS;
      S = S0 + m * SS;
      const float* const xm = m ? x + m * d.ms[0] : x;
      if (m) {
        model_params(d, params, m, pm);
        for (int i = 0; i < d.L * d.D * d.NPAR; ++i) {  // the gradient targets: dense per model, m parameter sizes on
          const int li = i / (d.D * d.NPAR), pi = i % d.NPAR;
          const size_t n = pi == 0 ? d.GH * (li == 0 ? (size_t)d.I : d.DH) : pi == 1 ? d.GH * d.H : d.GH;
          dpm[i] = dparams[i] ? dparams[i] + m * n : nullptr;
        }
      }
      const float* const* const params_m = m ? pm : params;
      float* const* const dparams_m = m ? dpm : dparams;
      float* const dxm = dx && m ? dx + m * d.TB * d.I : dx;
      const float* const ym = bp.y + m * mo.y;
      const float* const h0m = bp.h_0 ? bp.h_0 + m * mo.state : nullptr;
      const uint64_t* hdr = reinterpret_cast<const uint64_t*>(R);  // dropout seed/offset used by the forward

      // The gradient GEMMs of this layer: each runs on the tensor cores when it is eligible, on the FFMA GEMM otherwise.
      // The tensor cores need 16-byte aligned targets: a gradient view that is not (a caller's flat bucket behind an
      // odd-sized tensor) takes the FFMA GEMM instead of failing.
      const bool tc_l = tc_available() && (Il % 128 == 0);
      // layer input as seen by the forward GEMM; one split serves both directions. The padded steps of a ragged batch
      // have zero gate gradients, but 0 * NaN is NaN: layer 0's operand must be 0 there, not whatever the caller left in
      // x (the layers above read the recurrence's outputs, which are 0 past each length)
      GradSrc X{nullptr, simple_rows((long long)Il), TB, Il, S + sl.b_tc_x, false};
      if (l == 0 && fused_ln) {  // what the forward GEMM multiplied: LayerNorm(x), saved densely by the prologue (padding 0)
        X.p = R + rl.xln;
      } else if (l == 0 && lengths) {  // x with its padding zeroed, dense in the (unused without LayerNorm) b_dxln region
        rc = launch_valid_rows(xm, tb_rows(xs_t, xs_b, d.B), d.T, d.B, Il, lengths, S + sl.b_dxln, st);
        if (rc) return rc;
        X.p = S + sl.b_dxln;
      } else if (l == 0) {
        X.p = xm;
        X.rows = tb_rows(xs_t, xs_b, d.B);
      } else {
        X.p = layer_in ? layer_in[l - 1] : R + (drop ? rl.ydrop[l - 1] : rl.ylayer[l - 1]);
      }
      // dX_l goes to the caller's dx (layer 0) or to the dy of the layer below (scratch). With the fused LayerNorm the
      // layer-0 dgrad is d/dLN(x): it goes to scratch and through the LN backward below
      const bool ln_l0 = (l == 0) && fused_ln;
      const bool want_dx = (l > 0) || (dxm != nullptr) || (ln_l0 && (dln_gamma || dln_beta));
      float* Cx = S + sl.b_dy;
      RowMap cx_rows = simple_rows((long long)d.DH);
      if (ln_l0) {
        Cx = S + sl.b_dxln; cx_rows = simple_rows((long long)d.I);
      } else if (l == 0) {
        Cx = dxm; cx_rows = tb_rows(dxs_t, dxs_b, d.B);
      }
      const bool tc_dx = tc_l && want_dx && aligned_to(Cx, 16) && cx_rows.s_outer % 4 == 0 && cx_rows.s_inner % 4 == 0;
      for (int k = 0; k < d.D; ++k) {
        const float* const* pp = params_m + (size_t)(l * d.D + k) * d.NPAR;
        float* const* gp = dparams_m + (size_t)(l * d.D + k) * d.NPAR;
        float *dw_ih = gp[0], *dw_hh = gp[1], *db_ih = gp[2], *db_hh = gp[3];
        if (db_ih || db_hh) {
          rc = launch_bias_reduce(S + sl.b_bpart[k], bp.nslices_out, d.mode, d.H, db_ih, db_hh, accumulate, st);
          if (rc) return rc;
        }
        // this direction's operands (their split regions are reused by the next direction)
        GradSrc dG{S + sl.b_dgates[k], simple_rows(GH), TB, GH, S + sl.b_tc_dg, false};
        GradSrc dnr{S + sl.b_dghn[k], simple_rows(d.H), TB, d.H, S + sl.b_tc_hn, false};  // GRU: dn * r
        GradSrc h{ym + (long long)k * d.HO, tb_rows(bp.y_st, bp.y_sb, d.B), TB, d.HO, S + sl.b_tc_y, false};
        GradSrc w_ih{pp[0], simple_rows(Il), GH, Il, S + sl.b_tc_w, false};
        if (dw_ih) {  // dW_ih[GH, Il] = sum_tb dG[tb, :]^T X_l[tb, :]
          rc = run_grad_gemm({{&dG, 0, false}, {&X, 0, false}, GH, Il, TB, dw_ih, simple_rows(Il), accumulate, true,
                              tc_l && aligned_to(dw_ih, 16), "dW_ih"}, sl, S, tf32, st);
          if (rc) return rc;
        }
        if (dw_hh) {
          // dW_hh = sum_t dGh[t]^T h_{prev(t)}: rows are (t,b) flattened time-major, so the one-step shift is a row
          // offset of B (forward: dG[t] with h[t-1], t = 1..T-1; reverse: dG[t] with h[t+1], t = 0..T-2). LSTM, Elman:
          // one GEMM over all gates; GRU: the r,z rows from columns [0, 2H) of dG, the n rows from dn*r
          const int g0 = k == 0 ? d.B : 0, Kp = (d.T - 1) * d.B;
          // the tensor-core GEMM needs N = H a multiple of 128 (hidden sizes other than 128 / 256 may not be)
          const bool gru = d.mode == B200RNN_GRU,
                     tc = tc_l && aligned_to(dw_hh, 16) && d.T > 1 && d.P == 0 && d.HO % 128 == 0;
          rc = run_grad_gemm({{&dG, g0, false}, {&h, d.B - g0, false}, gru ? 2 * d.H : GH, d.HO, Kp, dw_hh,
                              simple_rows(d.HO), accumulate, true, tc, gru ? "dW_hh_rz" : "dW_hh"}, sl, S, tf32, st);
          if (rc) return rc;
          if (gru) {
            rc = run_grad_gemm({{&dnr, g0, false}, {&h, d.B - g0, false}, d.H, d.HO, Kp, dw_hh + (size_t)2 * d.H * d.HO,
                                simple_rows(d.HO), accumulate, true, tc, "dW_hh_n"}, sl, S, tf32, st);
            if (rc) return rc;
          }
        }
        if (dw_hh && h0m) {
          // the first scanned step's previous state is h_0: dW_hh += sum_b dGh[t_first(b), b]^T h_0[b]. The shifted GEMMs
          // above never pair that step with anything but a zero (T = 1: K = 0; ragged reverse rows: the masked output at
          // len_b), so nothing is counted twice. One fixed-order K = B FFMA GEMM: deterministic.
          GradSrc rows0{S + sl.b_h0, simple_rows(GH), d.B, GH, nullptr, false};  // [B][GH]
          GradSrc h0{h0m + (size_t)k * d.B * d.HO, simple_rows(d.HO), d.B, d.HO, nullptr, false};
          rc = launch_initial_state_rows(dG.p, dnr.p, d.mode, d.B, d.T, d.H, k == 1, lengths, S + sl.b_h0, st);
          if (rc) return rc;
          rc = run_grad_gemm({{&rows0, 0, false}, {&h0, 0, false}, GH, d.HO, d.B, dw_hh, simple_rows(d.HO), 1, false,
                              false, "dW_hh_h0"}, sl, S, tf32, st);
          if (rc) return rc;
        }
        if (d.P > 0 && gp[4]) {  // dW_hr[P, H] = sum_tb dh[tb, :]^T m[tb, :] (frozen and skipped steps have dh = 0)
          GradSrc dhp{S + sl.b_dhp[k], simple_rows(d.P), TB, d.P, nullptr, false};
          GradSrc m{R + rl.m[l][k], simple_rows(d.H), TB, d.H, nullptr, false};
          rc = run_grad_gemm({{&dhp, 0, false}, {&m, 0, false}, d.P, d.H, TB, gp[4], simple_rows(d.H), accumulate, true,
                              false, "dW_hr"}, sl, S, tf32, st);
          if (rc) return rc;
        }
        if (want_dx) {  // dX_l (+)= dG[TB, GH] W_ih[GH, Il]: dG read K-major, W_ih as it lies
          rc = run_grad_gemm({{&dG, 0, true}, {&w_ih, 0, false}, TB, Il, GH, Cx, cx_rows, k > 0, false, tc_dx, "dX"}, sl,
                             S, tf32, st);
          if (rc) return rc;
        }
      }
      if (l > 0 && drop) {  // gradient through the inter-layer dropout of layer l-1's output (same mask)
        rc = launch_dropout(S + sl.b_dy, S + sl.b_dy, d.TB * d.DH, d.p, hdr, (uint32_t)(l - 1), st);
        if (rc) return rc;
      }
      if (ln_l0 && want_dx) {  // LayerNorm backward: dx (caller's layout), dgamma, dbeta
        rc = launch_layernorm_bwd(xm, tb_rows(xs_t, xs_b, d.B), S + sl.b_dxln, (int)d.TB, d.I, ln_gamma, ln_eps, dxm,
                                  tb_rows(dxs_t, dxs_b, d.B), dln_gamma, dln_beta, accumulate, S + sl.b_lnpart, st,
                                  lengths, d.B);
        if (rc) return rc;
      }
    }
    R = R0;
    S = S0;
  }
  return B200RNN_OK;
}

// The backward of a 16-bit call: exact fp32 copies of every operand into the scratch behind the fp32 layout, the fp32
// backward on them (with the forward's fp32 top-layer output and rounded layer inputs from the reserve), then every
// gradient rounded once into the caller's 16-bit tensors (added to them with B200RNN_FLAG_ACCUMULATE_GRADS).
static int backward_h16(const b200rnn_desc* desc, const float* x, int64_t xs_t, int64_t xs_b, const float* const* params,
                        const float* dy, int64_t dys_t, int64_t dys_b, const float* dh_n, const float* dc_n,
                        const float* h_0, const float* c_0, float* dh_0, float* dc_0, const void* reserve,
                        void* scratch, float* dx, int64_t dxs_t, int64_t dxs_b, float* const* dparams,
                        const int32_t* lengths, void* stream_) {
  Dims d;
  int rc = check_desc(desc, &d);
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  if (d.B == 0 || d.T == 0) return B200RNN_OK;
  if (!x || !params || !dy || !reserve || !scratch || !dparams) {
    set_error("backward: null pointer argument");
    return B200RNN_ERR_INVALID;
  }
  if (!aligned_to(reserve, 256) || !aligned_to(scratch, 256)) {
    set_error("backward: reserve/scratch must be 256-byte aligned");
    return B200RNN_ERR_INVALID;
  }
  ReserveLayout rl;
  rc = make_reserve(d, &rl);
  if (rc) return rc;
  ScratchLayout sl;
  make_scratch(d, &sl);
  H16Scratch hs;
  make_h16_scratch(d, sl.b_total, &hs);
  const float* R = static_cast<const float*>(reserve);
  float* S = static_cast<float*>(scratch);
  const int dt = d.dt, TB = (int)d.TB, DH = (int)d.DH, nst = d.L * d.D * d.B;
  const RowMap hrows = simple_rows(d.H);
  rc = launch_widen16(x, tb_rows(xs_t, xs_b, d.B), TB, d.I, dt, S + hs.x32, st);
  if (!rc) rc = launch_widen16(dy, tb_rows(dys_t, dys_b, d.B), TB, DH, dt, S + hs.dy32, st);
  const float* src[4] = {dh_n, dc_n, h_0, c_0};
  const size_t at[4] = {hs.dhn, hs.dcn, hs.bh0, hs.bc0};
  const float* w[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int i = 0; i < 4 && !rc; ++i)
    if (src[i]) {
      rc = launch_widen16(src[i], hrows, nst, d.H, dt, S + at[i], st);
      w[i] = S + at[i];
    }
  if (rc) return rc;
  const float* p32[8 * 2 * 4];
  float* dp32[8 * 2 * 4];
  // fp32 master parameters: one launch rounds them into hs.w32 and the 16-bit weight_hh images
  const float* img[8 * 2 * 4];
  if (d.master) {
    rc = round_master_params(d, params, S, hs, true, true, img, st);
    if (rc) return rc;
  }
  for (int l = 0; l < d.L; ++l)
    for (int k = 0; k < d.D; ++k) {
      const int Il = l == 0 ? d.I : DH;
      const size_t n[4] = {d.GH * (size_t)Il, d.GH * (size_t)d.H, d.GH, d.GH};
      size_t off = 0;
      for (int i = 0; i < 4; ++i) {
        const size_t j = (size_t)(l * d.D + k) * 4 + i;
        if (!params[j]) {
          set_error("backward: null parameter pointer (layer %d dir %d)", l, k);
          return B200RNN_ERR_INVALID;
        }
        float* p = S + hs.w32[l][k] + off;
        if (!d.master) rc = launch_widen16(params[j], simple_rows((long long)n[i]), 1, (int)n[i], dt, p, st);
        if (rc) return rc;
        p32[j] = p;
        dp32[j] = dparams[j] ? S + hs.dw32[l][k] + off : nullptr;
        off += n[i];
      }
    }
  const float* layer_in[8];
  for (int l = 0; l + 1 < d.L; ++l) layer_in[l] = R + rl.xin[l];
  const void* whh16[8 * 2];
  for (int i = 0; i < d.L * d.D; ++i) whh16[i] = (d.master ? img : params)[(size_t)i * 4 + 1];
  b200rnn_desc d32 = *desc;
  // TF32 applies to fp32 calls only (forward_impl): the fp32 backward of a 16-bit call runs its 3xTF32 GEMMs
  d32.flags &= ~(B200RNN_FLAG_F16 | B200RNN_FLAG_BF16 | B200RNN_FLAG_ACCUMULATE_GRADS | B200RNN_FLAG_TF32 |
                 B200RNN_FLAG_F32_PARAMS);
  rc = backward_impl(&d32, S + hs.x32, (int64_t)d.B * d.I, d.I, p32, R + rl.ytop, (int64_t)d.B * DH, DH, S + hs.dy32,
                     (int64_t)d.B * DH, DH, nullptr, 0.f, w[0], w[1], reserve, scratch, dx ? S + hs.dx32 : nullptr,
                     (int64_t)d.B * d.I, d.I, dp32, lengths, nullptr, 0.f, nullptr, nullptr, w[2], w[3],
                     dh_0 ? S + hs.dh0 : nullptr, dc_0 ? S + hs.dc0 : nullptr, stream_, layer_in, dt, whh16);
  if (rc) return rc;
  const bool acc = (desc->flags & B200RNN_FLAG_ACCUMULATE_GRADS) != 0;
  if (dx) rc = launch_narrow16(S + hs.dx32, simple_rows(d.I), TB, d.I, dt, dx, tb_rows(dxs_t, dxs_b, d.B), false,
                               nullptr, st);
  if (!rc && dh_0) rc = launch_narrow16(S + hs.dh0, hrows, nst, d.H, dt, dh_0, hrows, false, nullptr, st);
  if (!rc && dc_0) rc = launch_narrow16(S + hs.dc0, hrows, nst, d.H, dt, dc_0, hrows, false, nullptr, st);
  if (!rc && d.master) {  // one launch: every gradient rounded to the 16-bit dtype and widened into its fp32 target
    Round16Seg seg[ROUND16_MAX_SEGS];
    int ns = 0;
    for (int l = 0; l < d.L; ++l)
      for (int k = 0; k < d.D; ++k) {
        const int Il = l == 0 ? d.I : DH;
        const size_t n[4] = {d.GH * (size_t)Il, d.GH * (size_t)d.H, d.GH, d.GH};
        for (int i = 0; i < 4; ++i) {
          const size_t j = (size_t)(l * d.D + k) * 4 + i;
          seg[ns++] = Round16Seg{dp32[j], nullptr, dparams[j], dparams[j] ? (long long)n[i] : 0};
        }
      }
    return launch_round16_multi(seg, ns, dt, acc ? ROUND16_GRAD_ADD : ROUND16_GRAD_SET, st);
  }
  for (int l = 0; l < d.L && !rc; ++l)
    for (int k = 0; k < d.D && !rc; ++k) {
      const int Il = l == 0 ? d.I : DH;
      const size_t n[4] = {d.GH * (size_t)Il, d.GH * (size_t)d.H, d.GH, d.GH};
      for (int i = 0; i < 4 && !rc; ++i) {
        const size_t j = (size_t)(l * d.D + k) * 4 + i;
        if (dparams[j])
          rc = launch_narrow16(dp32[j], simple_rows((long long)n[i]), 1, (int)n[i], dt, dparams[j],
                               simple_rows((long long)n[i]), acc, nullptr, st);
      }
    }
  return rc;
}

B200RNN_API int b200rnn_backward_fused(const b200rnn_desc* desc, const float* x, int64_t xs_t, int64_t xs_b,
                                       const float* const* params, const float* y, int64_t ys_t, int64_t ys_b,
                                       const float* dy, int64_t dys_t, int64_t dys_b, const float* dy_pool,
                                       float dy_pool_scale, const float* dh_n, const float* dc_n, const void* reserve,
                                       void* scratch, float* dx, int64_t dxs_t, int64_t dxs_b, float* const* dparams,
                                       const int32_t* lengths, const float* ln_gamma, float ln_eps, float* dln_gamma,
                                       float* dln_beta, void* stream_) {
  if (desc && desc_proj(desc) != 0) {
    set_error("backward_fused: the model-shell entry points do not take proj_size (use b200rnn_backward_hx)");
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (check_shell_desc(desc, "backward_fused")) return B200RNN_ERR_UNSUPPORTED;
  return backward_impl(desc, x, xs_t, xs_b, params, y, ys_t, ys_b, dy, dys_t, dys_b, dy_pool, dy_pool_scale, dh_n,
                       dc_n, reserve, scratch, dx, dxs_t, dxs_b, dparams, lengths, ln_gamma, ln_eps, dln_gamma,
                       dln_beta, nullptr, nullptr, nullptr, nullptr, stream_);
}

B200RNN_API int b200rnn_backward_hx(const b200rnn_desc* desc, const float* x, int64_t xs_t, int64_t xs_b,
                                    const float* const* params, const float* y, int64_t ys_t, int64_t ys_b,
                                    const float* dy, int64_t dys_t, int64_t dys_b, const float* dh_n,
                                    const float* dc_n, const float* h_0, const float* c_0, float* dh_0, float* dc_0,
                                    const void* reserve, void* scratch, float* dx, int64_t dxs_t, int64_t dxs_b,
                                    float* const* dparams, const int32_t* lengths, void* stream_) {
  Dims d;
  int rc = check_desc(desc, &d);
  if (rc) return rc;
  rc = check_initial_state(desc, h_0, c_0, dc_0, "backward_hx");
  if (rc) return rc;
  if (!dy) {
    set_error("backward: null pointer argument");
    return B200RNN_ERR_INVALID;
  }
  if (d.B > 0 && d.T == 0) {  // no step: the gradients pass from the final state to the initial one
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    const size_t es = d.dt ? 2 : sizeof(float);
    const size_t bytes[2] = {(size_t)d.L * d.D * d.B * d.HO * es, (size_t)d.L * d.D * d.B * d.H * es};
    const float* src[2] = {dh_n, dc_n};
    float* dst[2] = {dh_0, dc_0};
    for (int i = 0; i < 2; ++i) {
      if (!dst[i]) continue;
      if (src[i]) B200_CUDA_CHECK(cudaMemcpyAsync(dst[i], src[i], bytes[i], cudaMemcpyDeviceToDevice, st));
      else B200_CUDA_CHECK(cudaMemsetAsync(dst[i], 0, bytes[i], st));
    }
    return B200RNN_OK;
  }
  if (d.dt)
    return backward_h16(desc, x, xs_t, xs_b, params, dy, dys_t, dys_b, dh_n, dc_n, h_0, c_0, dh_0, dc_0, reserve,
                        scratch, dx, dxs_t, dxs_b, dparams, lengths, stream_);
  return backward_impl(desc, x, xs_t, xs_b, params, y, ys_t, ys_b, dy, dys_t, dys_b, nullptr, 0.f, dh_n, dc_n, reserve,
                       scratch, dx, dxs_t, dxs_b, dparams, lengths, nullptr, 0.f, nullptr, nullptr, h_0, c_0, dh_0, dc_0,
                       stream_);
}

B200RNN_API int b200rnn_backward(const b200rnn_desc* desc, const float* x, int64_t xs_t, int64_t xs_b,
                                 const float* const* params, const float* y, int64_t ys_t, int64_t ys_b,
                                 const float* dy, int64_t dys_t, int64_t dys_b, const float* dh_n,
                                 const float* dc_n, const void* reserve, void* scratch, float* dx, int64_t dxs_t,
                                 int64_t dxs_b, float* const* dparams, const int32_t* lengths, void* stream_) {
  if (!dy) {
    set_error("backward: null pointer argument");
    return B200RNN_ERR_INVALID;
  }
  if (desc && (desc->flags & (B200RNN_FLAG_F16 | B200RNN_FLAG_BF16)))
    return backward_h16(desc, x, xs_t, xs_b, params, dy, dys_t, dys_b, dh_n, dc_n, nullptr, nullptr, nullptr, nullptr,
                        reserve, scratch, dx, dxs_t, dxs_b, dparams, lengths, stream_);
  return backward_impl(desc, x, xs_t, xs_b, params, y, ys_t, ys_b, dy, dys_t, dys_b, nullptr, 0.f, dh_n, dc_n, reserve,
                       scratch, dx, dxs_t, dxs_b, dparams, lengths, nullptr, 0.f, nullptr, nullptr, nullptr, nullptr,
                       nullptr, nullptr, stream_);
}

// The descriptor of a tangent call: what forward mode does not run is refused before anything else
static int check_tangent_desc(const b200rnn_desc* desc, Dims* d) {
  if (desc && desc_proj(desc) != 0) {
    set_error("forward_tangent: proj_size is not supported in forward mode");
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (desc && (desc->flags & (B200RNN_FLAG_F16 | B200RNN_FLAG_BF16 | B200RNN_FLAG_F32_PARAMS))) {
    set_error("forward_tangent: forward mode is float32 only (no B200RNN_FLAG_F16 / _BF16 / _F32_PARAMS)");
    return B200RNN_ERR_UNSUPPORTED;
  }
  if (desc && (desc->flags & B200RNN_FLAG_FUSED_LN)) {
    set_error("forward_tangent: the model-shell fusions (B200RNN_FLAG_FUSED_LN) are not supported in forward mode");
    return B200RNN_ERR_UNSUPPORTED;
  }
  return check_desc(desc, d);
}

// Scratch of b200rnn_forward_tangent (floats): one tensor-core GEMM workspace shared by every GEMM of the call (they run
// one after the other on the stream), then per tangent direction its pre-activations (per layer direction [T,B,G*H]),
// the GRU's n-block h side ([T,B,H]) and the two buffers of an inner layer's tangent output ([T,B,D*H])
struct TangentLayout {
  size_t tc_ws, tc_ws_bytes;
  size_t pre[2], preh[2], ybuf[2];  // offsets within a direction's block
  size_t block, total;
};

static void make_tangent_layout(const Dims& d, TangentLayout* t) {
  const size_t g0 = gemm_tc_scratch_bytes((int)d.TB, (int)d.GH, d.I);
  const size_t g1 = gemm_tc_scratch_bytes((int)d.TB, (int)d.GH, (int)d.DH);
  t->tc_ws_bytes = g0 > g1 ? g0 : g1;
  t->tc_ws = 0;
  size_t off = 0;
  for (int k = 0; k < 2; ++k) {
    t->pre[k] = off;
    if (k < d.D) off += align_up(d.TB * d.GH, ALIGN_F);
  }
  for (int k = 0; k < 2; ++k) {
    t->preh[k] = off;
    if (k < d.D && d.mode == B200RNN_GRU) off += align_up(d.TB * (size_t)d.H, ALIGN_F);
  }
  for (int k = 0; k < 2; ++k) {
    t->ybuf[k] = off;
    if (d.L > 1) off += align_up(d.TB * d.DH, ALIGN_F);
  }
  t->block = off;
  t->total = align_up(t->tc_ws_bytes / sizeof(float) + 1, ALIGN_F) + (size_t)d.M * t->block;
}

B200RNN_API int b200rnn_tangent_workspace_bytes(const b200rnn_desc* desc, size_t* scratch_bytes) {
  Dims d;
  const int rc = check_tangent_desc(desc, &d);
  if (rc) return rc;
  TangentLayout tl;
  make_tangent_layout(d, &tl);
  if (scratch_bytes) *scratch_bytes = tl.total * sizeof(float);
  return B200RNN_OK;
}

// Forward-mode AD of a saving forward (include/b200rnn.h). Per layer and direction: the tangent pre-activations by the
// time-parallel GEMMs, W_ih x' + W_ih' x (+ W_hh' h_{t-1}, the primal output shifted by one step and h_0 for the first
// step), then one tangent recurrence launch for every direction of the layer and every tangent direction, then the
// primal's dropout mask on an inner layer's tangent output, which is the next layer's x'.
B200RNN_API int b200rnn_forward_tangent(const b200rnn_desc* desc, const float* x, int64_t xs_t, int64_t xs_b,
                                        const float* const* params, const float* y, int64_t ys_t, int64_t ys_b,
                                        const float* h_0, const float* c_0, const void* reserve,
                                        const int32_t* lengths, const float* x_dot, const float* const* params_dot,
                                        const float* h_0_dot, const float* c_0_dot, float* y_dot, int64_t yds_t,
                                        int64_t yds_b, float* h_n_dot, float* c_n_dot, void* scratch, void* stream_) {
  if (lengths) {
    set_error("forward_tangent: ragged batches (lengths) are not supported in forward mode");
    return B200RNN_ERR_UNSUPPORTED;
  }
  Dims d;
  int rc = check_tangent_desc(desc, &d);
  if (rc) return rc;
  rc = check_initial_state(desc, h_0, c_0, c_0_dot, "forward_tangent");
  if (rc) return rc;
  // an output with no element may be NULL (an empty tensor's data pointer): y_dot when B == 0 or T == 0, the states'
  // tangents when B == 0
  const bool empty = d.B == 0 || d.T == 0, lstm = d.mode == B200RNN_LSTM;
  if ((!empty && !y_dot) || (d.B > 0 && (!h_n_dot || (lstm && !c_n_dot))) || (!lstm && c_n_dot)) {
    set_error("forward_tangent: y_dot and h_n_dot (and, for the LSTM only, c_n_dot) are required");
    return B200RNN_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const int M = d.M;  // tangent directions
  const size_t nstate = (size_t)d.L * d.D * d.B * d.H;
  if (empty) {  // no step: the final state's tangent is the initial one's
    if (nstate == 0) return B200RNN_OK;
    if (h_0_dot) B200_CUDA_CHECK(cudaMemcpyAsync(h_n_dot, h_0_dot, M * nstate * sizeof(float), cudaMemcpyDeviceToDevice, st));
    else B200_CUDA_CHECK(cudaMemsetAsync(h_n_dot, 0, M * nstate * sizeof(float), st));
    if (c_n_dot) {
      if (c_0_dot) B200_CUDA_CHECK(cudaMemcpyAsync(c_n_dot, c_0_dot, M * nstate * sizeof(float), cudaMemcpyDeviceToDevice, st));
      else B200_CUDA_CHECK(cudaMemsetAsync(c_n_dot, 0, M * nstate * sizeof(float), st));
    }
    return B200RNN_OK;
  }
  if (!x || !params || !y || !reserve || !scratch) {
    set_error("forward_tangent: null pointer argument");
    return B200RNN_ERR_INVALID;
  }
  if (!aligned_to(reserve, 256) || !aligned_to(scratch, 256)) {
    set_error("forward_tangent: reserve/scratch must be 256-byte aligned");
    return B200RNN_ERR_INVALID;
  }
  for (int i = 0; i < d.L * d.D * 4; ++i)
    if (!params[i]) {
      set_error("forward_tangent: null parameter pointer (index %d)", i);
      return B200RNN_ERR_INVALID;
    }
  ReserveLayout rl;
  rc = make_reserve(d, &rl);
  if (rc) return rc;
  TangentLayout tl;
  make_tangent_layout(d, &tl);
  const float* R = static_cast<const float*>(reserve);
  float* const tc_ws = static_cast<float*>(scratch);
  float* const S0 = tc_ws + align_up(tl.tc_ws_bytes / sizeof(float) + 1, ALIGN_F);  // direction 0's block
  const size_t SS = tl.block;
  const uint64_t* hdr = reinterpret_cast<const uint64_t*>(R);  // the primal's dropout seed / offset
  const bool drop = d.training && d.p > 0.f && d.L > 1;
  const bool tf32 = (desc->flags & B200RNN_FLAG_TF32) != 0;
  const int TB = (int)d.TB, GH = (int)d.GH, H = d.H;
  const bool gru = d.mode == B200RNN_GRU;
  // an inner layer's tangent output, per tangent direction: two buffers of its block, layer l writing l & 1
  const size_t* ybuf = tl.ybuf;
  // C (+)= A W^T over the FFMA GEMM; `tc_ok`: the first (writing) GEMM of a buffer may take the tensor cores
  auto gemm = [&](const float* A, RowMap a_rows, const float* W, float* C, int Mr, int N, int K, RowMap c_rows, int acc,
                  bool tc_ok) {
    GemmParams g;
    memset(&g, 0, sizeof(g));
    g.A = A; g.a_rows = a_rows; g.a_kcontig = 1;
    g.B = W; g.b_rows = simple_rows(K); g.b_kcontig = 1;
    g.C = C; g.c_rows = c_rows;
    g.M = Mr; g.N = N; g.K = K;
    g.accumulate = acc;
    if (tc_ok && tc_available()) {
      g.tc_ws = tc_ws;
      g.tc_ws_bytes = tl.tc_ws_bytes;
      g.tc_tf32 = tf32 ? 1 : 0;
    }
    return launch_gemm(g, nullptr, 0, st);
  };
  for (int l = 0; l < d.L; ++l) {
    const int Il = l == 0 ? d.I : (int)d.DH;
    const bool top = l == d.L - 1;
    // the primal layer input and output, as the forward read and wrote them
    const float* in = l == 0 ? x : R + (drop ? rl.ydrop[l - 1] : rl.ylayer[l - 1]);
    const RowMap in_rows = l == 0 ? tb_rows(xs_t, xs_b, d.B) : simple_rows((long long)d.DH);
    const float* out = top ? y : R + rl.ylayer[l];
    const long long out_st = top ? ys_t : (long long)d.B * d.DH, out_sb = top ? ys_b : (long long)d.DH;
    RecTanParams rp;
    memset(&rp, 0, sizeof(rp));
    rp.mode = d.mode; rp.B = d.B; rp.T = d.T; rp.H = H; rp.D = d.D;
    rp.y = out; rp.y_st = out_st; rp.y_sb = out_sb;
    rp.h_0 = h_0 ? h_0 + (size_t)l * d.D * d.B * H : nullptr;
    rp.c_0 = c_0 ? c_0 + (size_t)l * d.D * d.B * H : nullptr;
    for (int m = 0; m < M; ++m) {
      float* const S = S0 + m * SS;
      // the tangent layer input x' (layer 0: the caller's dense [T,B,I] block, NULL = 0)
      const float* in_dot = l == 0 ? (x_dot ? x_dot + (size_t)m * TB * d.I : nullptr) : S + ybuf[(l - 1) & 1];
      for (int k = 0; k < d.D; ++k) {
        const size_t pi = (size_t)(l * d.D + k) * 4;
        const float* const* pp = params + pi;
        const float* wih_d = params_dot && params_dot[pi] ? params_dot[pi] + (size_t)m * GH * Il : nullptr;
        const float* whh_d = params_dot && params_dot[pi + 1] ? params_dot[pi + 1] + (size_t)m * GH * H : nullptr;
        float* pre = S + tl.pre[k];
        float* preh = S + tl.preh[k];
        bool pre_init = false;
        if (in_dot) {  // W_ih x'
          rc = gemm(in_dot, simple_rows(Il), pp[0], pre, TB, GH, Il, simple_rows(GH), 0, true);
          if (rc) return rc;
          pre_init = true;
        }
        if (wih_d) {  // W_ih' x
          rc = gemm(in, in_rows, wih_d, pre, TB, GH, Il, simple_rows(GH), pre_init, !pre_init);
          if (rc) return rc;
          pre_init = true;
        }
        if (whh_d) {
          // W_hh' h_{t-1}: the primal output one step back (reverse: one step ahead) for every step but the first, h_0
          // (or nothing) for the first. GRU: the r, z blocks into pre, the n block into preh (r multiplies it)
          if (!pre_init) B200_CUDA_CHECK(cudaMemsetAsync(pre, 0, d.TB * d.GH * sizeof(float), st));
          if (gru) B200_CUDA_CHECK(cudaMemsetAsync(preh, 0, d.TB * H * sizeof(float), st));
          pre_init = true;
          const float* hp = out + (long long)k * H + (k == 0 ? 0 : out_st);
          const size_t c_row0 = k == 0 ? (size_t)d.B : 0;  // first C row the shifted GEMM writes
          const int Mr = (d.T - 1) * d.B, nrz = gru ? 2 * H : GH;
          const RowMap hp_rows = tb_rows(out_st, out_sb, d.B);
          const float* h0k = rp.h_0 ? rp.h_0 + (size_t)k * d.B * H : nullptr;
          const size_t first = (size_t)(k == 0 ? 0 : d.T - 1) * d.B;  // rows of the first scanned step
          rc = gemm(hp, hp_rows, whh_d, pre + c_row0 * GH, Mr, nrz, H, simple_rows(GH), 1, false);
          if (!rc && h0k) rc = gemm(h0k, simple_rows(H), whh_d, pre + first * GH, d.B, nrz, H, simple_rows(GH), 1, false);
          if (!rc && gru) {
            rc = gemm(hp, hp_rows, whh_d + (size_t)2 * H * H, preh + c_row0 * H, Mr, H, H, simple_rows(H), 1, false);
            if (!rc && h0k)
              rc = gemm(h0k, simple_rows(H), whh_d + (size_t)2 * H * H, preh + first * H, d.B, H, H, simple_rows(H), 1, false);
          }
          if (rc) return rc;
        }
        if (m > 0) continue;  // the launch takes direction 0's pointers and the strides below
        rp.w_hh[k] = pp[1];
        rp.gates[k] = R + rl.gates[l][k];
        rp.extra[k] = is_elman(d.mode) ? nullptr : R + rl.extra[l][k];
        rp.pre[k] = pre_init ? pre : nullptr;
        rp.preh[k] = gru && whh_d ? preh : nullptr;
        rp.bih_dot[k] = params_dot ? params_dot[pi + 2] : nullptr;
        rp.bhh_dot[k] = params_dot ? params_dot[pi + 3] : nullptr;
      }
    }
    rp.h0_dot = h_0_dot ? h_0_dot + (size_t)l * d.D * d.B * H : nullptr;
    rp.c0_dot = c_0_dot ? c_0_dot + (size_t)l * d.D * d.B * H : nullptr;
    if (top) {
      rp.ydot = y_dot; rp.yd_st = yds_t; rp.yd_sb = yds_b; rp.m_ydot = (long long)(d.TB * d.DH);
    } else {
      rp.ydot = S0 + ybuf[l & 1]; rp.yd_st = (long long)d.B * d.DH; rp.yd_sb = (long long)d.DH; rp.m_ydot = (long long)SS;
    }
    rp.hn_dot = h_n_dot + (size_t)l * d.D * d.B * H;
    rp.cn_dot = c_n_dot ? c_n_dot + (size_t)l * d.D * d.B * H : nullptr;
    rp.m_pre = rp.m_preh = (long long)SS;
    rp.m_bdot = GH;
    rp.m_state = (long long)nstate;
    rc = launch_rec_tangent(rp, M, st);
    if (rc) return rc;
    if (drop && !top)  // the primal's mask (same header, same stream id) on the tangent: the next layer's x'
      for (int m = 0; m < M; ++m) {
        float* yd = S0 + m * SS + ybuf[l & 1];
        rc = launch_dropout(yd, yd, d.TB * d.DH, d.p, hdr, (uint32_t)l, st);
        if (rc) return rc;
      }
  }
  return B200RNN_OK;
}

B200RNN_API int b200rnn_cell_workspace_bytes(const b200rnn_cell_desc* desc, size_t* saved_bytes, size_t* scratch_bytes) {
  CellDims d;
  const int rc = check_cell_desc(desc, &d);
  if (rc) return rc;
  CellSaved sv;
  make_cell_saved(d, &sv);
  CellScratch sc;
  make_cell_scratch(d, &sc);
  if (saved_bytes) *saved_bytes = sv.total * sizeof(float);
  if (scratch_bytes) *scratch_bytes = sc.total * sizeof(float);
  return B200RNN_OK;
}

// x_ld / h_ld / c_ld of a cell call: rows must not overlap (a single row may have any stride)
static bool cell_rows_ok(int B, int64_t ld, int width) { return B <= 1 || ld >= width; }

// params: 4 pointers (weights required, biases NULL exactly when the descriptor says NO_BIAS)
static int check_cell_params(const CellDims& d, const float* const* params, const char* what) {
  if (!params || !params[0] || !params[1]) {
    set_error("%s: null weight pointer", what);
    return B200RNN_ERR_INVALID;
  }
  if ((params[2] != nullptr) != d.bias || (params[3] != nullptr) != d.bias) {
    set_error("%s: bias pointers must be both set, or both NULL with B200RNN_FLAG_NO_BIAS", what);
    return B200RNN_ERR_INVALID;
  }
  return B200RNN_OK;
}

B200RNN_API int b200rnn_cell_forward(const b200rnn_cell_desc* desc, const float* x, int64_t x_ld, const float* h,
                                     int64_t h_ld, const float* c, int64_t c_ld, const float* const* params,
                                     float* h_out, float* c_out, void* saved, void* stream_) {
  CellDims d;
  int rc = check_cell_desc(desc, &d);
  if (rc) return rc;
  const bool lstm = d.mode == B200RNN_LSTM;
  if (!lstm && (c || c_out)) {
    set_error("cell_forward: a %s cell has no cell state (c / c_out must be NULL)", mode_name(d.mode));
    return B200RNN_ERR_INVALID;
  }
  if (d.B == 0) return B200RNN_OK;
  if (!x || !h_out || (lstm && !c_out)) {
    set_error("cell_forward: null pointer argument");
    return B200RNN_ERR_INVALID;
  }
  rc = check_cell_params(d, params, "cell_forward");
  if (rc) return rc;
  if (!cell_rows_ok(d.B, x_ld, d.I) || (h && !cell_rows_ok(d.B, h_ld, d.H)) || (c && !cell_rows_ok(d.B, c_ld, d.H))) {
    set_error("cell_forward: a row stride is smaller than its row (x_ld=%lld h_ld=%lld c_ld=%lld)", (long long)x_ld,
              (long long)h_ld, (long long)c_ld);
    return B200RNN_ERR_INVALID;
  }
  if (d.save && (!saved || !aligned_to(saved, 256))) {
    set_error("cell_forward: B200RNN_FLAG_SAVE_FOR_BACKWARD needs a 256-byte aligned saved-state buffer");
    return B200RNN_ERR_INVALID;
  }
  CellSaved sv;
  make_cell_saved(d, &sv);
  float* SV = static_cast<float*>(saved);
  CellFwdParams p;
  memset(&p, 0, sizeof(p));
  p.mode = d.mode; p.B = d.B; p.I = d.I; p.H = d.H;
  p.tf32 = d.tf32 ? 1 : 0;
  p.x = x; p.x_ld = x_ld;
  p.h = h; p.h_ld = h_ld;
  p.c = c; p.c_ld = c_ld;
  p.w_ih = params[0]; p.w_hh = params[1]; p.b_ih = params[2]; p.b_hh = params[3];
  p.h_out = h_out; p.c_out = c_out;
  p.gates = d.save ? SV + sv.gates : nullptr;
  p.extra = d.save && !is_elman(d.mode) ? SV + sv.extra : nullptr;
  return launch_cell_fwd(p, static_cast<cudaStream_t>(stream_));
}

B200RNN_API int b200rnn_cell_backward(const b200rnn_cell_desc* desc, const float* x, int64_t x_ld, const float* h,
                                      int64_t h_ld, const float* c, int64_t c_ld, const float* const* params,
                                      const float* dh_out, const float* dc_out, const void* saved, float* dx,
                                      float* dh, float* dc, float* const* dparams, void* scratch, void* stream_) {
  CellDims d;
  int rc = check_cell_desc(desc, &d);
  if (rc) return rc;
  const bool lstm = d.mode == B200RNN_LSTM;
  if (!lstm && (c || dc_out || dc)) {
    set_error("cell_backward: a %s cell has no cell state (c / dc_out / dc must be NULL)", mode_name(d.mode));
    return B200RNN_ERR_INVALID;
  }
  if (!dparams) {
    set_error("cell_backward: null pointer argument");
    return B200RNN_ERR_INVALID;
  }
  if (!d.bias && (dparams[2] || dparams[3])) {
    set_error("cell_backward: bias gradients requested with B200RNN_FLAG_NO_BIAS");
    return B200RNN_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const size_t GH = d.GH;
  const size_t nparam[4] = {GH * d.I, GH * d.H, GH, GH};
  if (d.B == 0) {  // no row: the parameter gradients are zero
    if (!d.accumulate)
      for (int i = 0; i < 4; ++i)
        if (dparams[i]) B200_CUDA_CHECK(cudaMemsetAsync(dparams[i], 0, nparam[i] * sizeof(float), st));
    return B200RNN_OK;
  }
  if (!x || !saved || !scratch) {
    set_error("cell_backward: null pointer argument");
    return B200RNN_ERR_INVALID;
  }
  rc = check_cell_params(d, params, "cell_backward");
  if (rc) return rc;
  if (!cell_rows_ok(d.B, x_ld, d.I) || (h && !cell_rows_ok(d.B, h_ld, d.H)) || (c && !cell_rows_ok(d.B, c_ld, d.H))) {
    set_error("cell_backward: a row stride is smaller than its row (x_ld=%lld h_ld=%lld c_ld=%lld)", (long long)x_ld,
              (long long)h_ld, (long long)c_ld);
    return B200RNN_ERR_INVALID;
  }
  if (!aligned_to(saved, 256) || !aligned_to(scratch, 256)) {
    set_error("cell_backward: saved / scratch must be 256-byte aligned");
    return B200RNN_ERR_INVALID;
  }
  CellSaved sv;
  make_cell_saved(d, &sv);
  CellScratch sc;
  make_cell_scratch(d, &sc);
  const float* SV = static_cast<const float*>(saved);
  float* S = static_cast<float*>(scratch);
  const int accumulate = d.accumulate ? 1 : 0;
  const int B = d.B, I = d.I, H = d.H, G = (int)GH;

  // gate gradients; GRU: dh = z * dh' + dG_h W_hh, the direct term goes to dh first; LSTM: dc is final here; Elman:
  // dh = dpre W_hh, no direct term
  CellBwdParams bp;
  memset(&bp, 0, sizeof(bp));
  bp.mode = d.mode; bp.B = B; bp.H = H;
  const bool elman = is_elman(d.mode);
  bp.gates = SV + sv.gates; bp.extra = elman ? nullptr : SV + sv.extra;
  bp.h = h; bp.h_ld = h_ld;
  bp.c = c; bp.c_ld = c_ld;
  bp.dh_out = dh_out; bp.dc_out = dc_out;
  bp.dg_x = S + sc.dgx;
  bp.dg_h = d.mode == B200RNN_GRU ? S + sc.dgh : nullptr;
  bp.direct = lstm ? dc : elman ? nullptr : dh;
  bp.part = S + sc.part;
  rc = launch_cell_bwd(bp, st);
  if (rc) return rc;
  if (dparams[2] || dparams[3]) {
    rc = launch_bias_reduce(bp.part, cell_bwd_slices(B), d.mode, H, dparams[2], dparams[3], accumulate, st);
    if (rc) return rc;
  }

  // the gradient GEMMs, as the sequence backward runs them (run_grad_gemm: tensor cores where eligible, else FFMA)
  const bool tc_x = d.tc_x && tc_available(), tc_h = d.tc_h && tc_available();
  GradSrc DGX{S + sc.dgx, simple_rows(G), B, G, S + sc.tc_dgx, false};
  GradSrc DGH_gru{S + sc.dgh, simple_rows(G), B, G, S + sc.tc_dgh, false};
  GradSrc& DGH = d.mode == B200RNN_GRU ? DGH_gru : DGX;  // LSTM, Elman: the h-part gate gradients are the x-part ones
  GradSrc X{x, simple_rows(x_ld), B, I, S + sc.tc_x, false};
  GradSrc Hs{h, simple_rows(h_ld), B, H, S + sc.tc_h, false};
  GradSrc WIH{params[0], simple_rows(I), G, I, S + sc.tc_wih, false};
  GradSrc WHH{params[1], simple_rows(H), G, H, S + sc.tc_whh, false};
  const ScratchLayout& sl = sc.gemm;
  if (dparams[0]) {  // dW_ih [GH, I] = dG_x^T x
    rc = run_grad_gemm({{&DGX, 0, false}, {&X, 0, false}, G, I, B, dparams[0], simple_rows(I), accumulate, true,
                        tc_x && aligned_to(dparams[0], 16), "cell dW_ih"}, sl, S, d.tf32, st);
    if (rc) return rc;
  }
  if (dparams[1] && h) {  // dW_hh [GH, H] = dG_h^T h
    rc = run_grad_gemm({{&DGH, 0, false}, {&Hs, 0, false}, G, H, B, dparams[1], simple_rows(H), accumulate, true,
                        tc_h && aligned_to(dparams[1], 16), "cell dW_hh"}, sl, S, d.tf32, st);
    if (rc) return rc;
  } else if (dparams[1] && !accumulate) {  // h = 0: nothing reaches W_hh
    B200_CUDA_CHECK(cudaMemsetAsync(dparams[1], 0, nparam[1] * sizeof(float), st));
  }
  if (dx) {  // dx [B, I] = dG_x W_ih
    rc = run_grad_gemm({{&DGX, 0, true}, {&WIH, 0, false}, B, I, G, dx, simple_rows(I), 0, false,
                        tc_x && aligned_to(dx, 16), "cell dx"}, sl, S, d.tf32, st);
    if (rc) return rc;
  }
  if (dh) {  // dh [B, H] (+)= dG_h W_hh
    const int acc_dh = d.mode == B200RNN_GRU ? 1 : 0;  // the GRU's direct term z * dh' is in dh already
    rc = run_grad_gemm({{&DGH, 0, true}, {&WHH, 0, false}, B, H, G, dh, simple_rows(H), acc_dh, false,
                        tc_h && aligned_to(dh, 16), "cell dh"}, sl, S, d.tf32, st);
    if (rc) return rc;
  }
  return B200RNN_OK;
}

B200RNN_API int b200rnn_gemm_f32(int M, int N, int K, const float* A, int64_t lda, int a_kcontig, const float* B,
                     int64_t ldb, int b_kcontig, float* C, int64_t ldc, const float* bias, int accumulate,
                     void* scratch, size_t scratch_bytes, void* stream_) {
  if (M < 0 || N < 0 || K < 0) {
    set_error("gemm: negative dimension");
    return B200RNN_ERR_INVALID;
  }
  GemmParams g;
  memset(&g, 0, sizeof(g));
  g.A = A; g.a_rows = simple_rows(lda); g.a_kcontig = a_kcontig;
  g.B = B; g.b_rows = simple_rows(ldb); g.b_kcontig = b_kcontig;
  g.C = C; g.c_rows = simple_rows(ldc);
  g.M = M; g.N = N; g.K = K;
  g.bias1 = bias;
  g.accumulate = accumulate;
  g.tc_ws = scratch;  // used by the tensor-core 3xTF32 path when the problem is eligible and the buffer is large enough
  g.tc_ws_bytes = scratch_bytes;
  return launch_gemm(g, scratch, scratch_bytes, static_cast<cudaStream_t>(stream_));
}

/* test only (not declared in the public header): the input projection's fp32-A tensor-core GEMM as the forward runs
   it, C[M][N] = A W^T + bias. Row m = t * a_batch + b of A sits at A + t * a_st + b * a_sb (a_batch = 0: dense rows,
   a_st floats apart) and is read in place; W [N][K] is split into `scratch` per call. ready != NULL: streamed launch
   on stream_clusters 4-CTA clusters, the M / 128 counters must be zero on entry. */
B200RNN_API int b200rnn_debug_gemm_f32a(int M, int N, int K, const float* A, int64_t a_st, int64_t a_sb, int a_batch,
                                        const float* W, float* C, const float* bias, int* ready, int stream_clusters,
                                        void* scratch, size_t scratch_bytes, void* stream_) {
  GemmParams g;
  memset(&g, 0, sizeof(g));
  g.A = A; g.a_rows = a_batch > 0 ? tb_rows(a_st, a_sb, a_batch) : simple_rows(a_st); g.a_kcontig = 1;
  g.B = W; g.b_rows = simple_rows(K); g.b_kcontig = 1;
  g.C = C; g.c_rows = simple_rows(N);
  g.M = M; g.N = N; g.K = K;
  g.bias1 = bias;
  g.tc_a_f32 = 1;
  g.tc_ready = ready;
  g.tc_stream_clusters = stream_clusters;
  if (!gemm_tc_eligible(g, scratch_bytes) || !tc_a_f32_in_place(A, g.a_rows, M, K)) {
    set_error("debug_gemm_f32a: problem not eligible for the fp32-A tensor-core path");
    return B200RNN_ERR_UNSUPPORTED;
  }
  return launch_gemm_tc(g, scratch, scratch_bytes, static_cast<cudaStream_t>(stream_));
}

/* test only (not declared in the public header): the no-grad forward's fp16-pair input projection, arguments as
   b200rnn_debug_gemm_f32a (W split into fp16 pairs in `scratch` per call); N % 128 == 0 and K % 64 == 0 */
B200RNN_API int b200rnn_debug_gemm_f16a(int M, int N, int K, const float* A, int64_t a_st, int64_t a_sb, int a_batch,
                                        const float* W, float* C, const float* bias, int* ready, int stream_clusters,
                                        void* scratch, size_t scratch_bytes, void* stream_) {
  GemmParams g;
  memset(&g, 0, sizeof(g));
  g.A = A; g.a_rows = a_batch > 0 ? tb_rows(a_st, a_sb, a_batch) : simple_rows(a_st); g.a_kcontig = 1;
  g.B = W; g.b_rows = simple_rows(K); g.b_kcontig = 1;
  g.C = C; g.c_rows = simple_rows(N);
  g.M = M; g.N = N; g.K = K;
  g.bias1 = bias;
  g.tc_a_f32 = 1;
  g.tc_h16 = 1;
  g.tc_ready = ready;
  g.tc_stream_clusters = stream_clusters;
  if (!g16::shape_ok(N, K) || !gemm_tc_eligible(g, scratch_bytes) || !tc_a_f32_in_place(A, g.a_rows, M, K)) {
    set_error("debug_gemm_f16a: problem not eligible for the fp16-pair tensor-core path");
    return B200RNN_ERR_UNSUPPORTED;
  }
  return launch_gemm_tc(g, scratch, scratch_bytes, static_cast<cudaStream_t>(stream_));
}

/* test only (not declared in the public header): gradient GEMMs as the backward runs them, through run_grad_gemm,
   in order, over shared sources (a source is split for the tensor cores by the first GEMM that reads it).
   srcs: nsrc rows of 6 int64 {pointer, s_outer, s_inner, inner_n, R, C}: an fp32 [R][C], row r at pointer +
   s_outer * (r / inner_n) + s_inner * (r % inner_n) floats.
   gemms: ngemm rows of 16 int64 {a_src, a_row0, a_kcontig, b_src, b_row0, b_kcontig, M, N, K, C pointer, c_s_outer,
   c_s_inner, c_inner_n, accumulate, splitk, tc}. tf32: single-pass TF32 tensor-core GEMMs (B200RNN_FLAG_TF32).
   The scratch is laid out as the backward's: split-K workspaces of the backward's sizes, one split region per source.
   scratch == NULL: *scratch_bytes receives the size needed. plans (optional): per GEMM the split count and its chunk
   (k-blocks of 32 on the tensor cores, K values on FFMA) the launch ran with. */
B200RNN_API int b200rnn_debug_grad_gemm(const int64_t* srcs, int nsrc, const int64_t* gemms, int ngemm, int tf32,
                                        void* scratch, size_t* scratch_bytes, int* plans, void* stream_) {
  constexpr int MAX_SRC = 16;
  if (!srcs || !gemms || !scratch_bytes || nsrc < 1 || nsrc > MAX_SRC || ngemm < 0) {
    set_error("debug_grad_gemm: bad arguments");
    return B200RNN_ERR_INVALID;
  }
  GradSrc src[MAX_SRC];
  size_t gb = 0, off = 0;
  for (int j = 0; j < ngemm; ++j) {  // the FFMA split-K workspace: the backward's formula, largest over the GEMMs
    const int64_t* q = gemms + (size_t)j * 16;
    if (q[14] && !q[15]) {
      const size_t b = gemm_scratch_bytes((int)q[6], (int)q[7], (int)q[8]);
      gb = b > gb ? b : gb;
    }
  }
  ScratchLayout sl;
  memset(&sl, 0, sizeof(sl));
  sl.b_gemm = off;
  sl.b_gemm_bytes = gb;
  off += align_up(gb / sizeof(float) + 1, ALIGN_F);
  size_t split_off[MAX_SRC];
  for (int i = 0; i < nsrc; ++i) {
    const int64_t* q = srcs + (size_t)i * 6;
    if (!q[0] || q[3] < 1 || q[4] < 1 || q[5] < 1) {
      set_error("debug_grad_gemm: source %d: null pointer or empty shape", i);
      return B200RNN_ERR_INVALID;
    }
    src[i] = GradSrc{reinterpret_cast<const float*>(q[0]), RowMap{q[1], q[2], (int)q[3]}, (int)q[4], (int)q[5],
                     nullptr, false};
    split_off[i] = off;
    off += align_up(2 * (size_t)q[4] * q[5], ALIGN_F);
  }
  sl.b_tc_part = off;
  sl.b_tc_part_bytes = TC_PART_BYTES;
  off += align_up(TC_PART_BYTES / sizeof(float), ALIGN_F);
  if (!scratch) {
    *scratch_bytes = off * sizeof(float);
    return B200RNN_OK;
  }
  if (*scratch_bytes < off * sizeof(float) || !aligned_to(scratch, 256)) {
    set_error("debug_grad_gemm: the scratch must be 256-byte aligned and hold %zu bytes", off * sizeof(float));
    return B200RNN_ERR_INVALID;
  }
  float* S = static_cast<float*>(scratch);
  for (int i = 0; i < nsrc; ++i) src[i].split = S + split_off[i];
  for (int j = 0; j < ngemm; ++j) {
    const int64_t* q = gemms + (size_t)j * 16;
    GradGemm g{{nullptr, (int)q[1], q[2] != 0}, {nullptr, (int)q[4], q[5] != 0}, (int)q[6], (int)q[7], (int)q[8],
               reinterpret_cast<float*>(q[9]), RowMap{q[10], q[11], (int)q[12]}, (int)q[13], q[14] != 0, q[15] != 0,
               "debug"};
    // every access stays inside the sources: a kcontig operand reads rows [row0, row0 + M or N) and columns [0, K),
    // the others rows [row0, row0 + K) and columns [0, M or N); a row offset must keep the row map linear
    for (int o = 0; o < 2; ++o) {
      GradOperand& op = o ? g.b : g.a;
      const int si = (int)(o ? q[3] : q[0]), mn = o ? g.N : g.M;
      if (si < 0 || si >= nsrc) {
        set_error("debug_grad_gemm: gemm %d: no source %d", j, si);
        return B200RNN_ERR_INVALID;
      }
      op.src = &src[si];
      const GradSrc& s = src[si];
      const int rows = op.kcontig ? mn : g.K, cols = op.kcontig ? g.K : mn;
      const bool linear = s.rows.inner_n >= s.R || op.row0 % s.rows.inner_n == 0;
      if (op.row0 < 0 || (long long)op.row0 + rows > s.R || cols > s.C || !linear || (g.tc && s.C % 4 != 0)) {
        set_error("debug_grad_gemm: gemm %d operand %d does not fit source %d", j, o, si);
        return B200RNN_ERR_INVALID;
      }
    }
    if (g.M < 1 || g.N < 1 || g.K < 1 || !g.C || g.c_rows.inner_n < 1) {
      set_error("debug_grad_gemm: gemm %d: bad shape or output", j);
      return B200RNN_ERR_INVALID;
    }
    GradPlan p;
    const int rc = run_grad_gemm(g, sl, S, tf32 != 0, static_cast<cudaStream_t>(stream_), &p);
    if (rc) return rc;
    if (plans) {
      plans[2 * j] = p.splitk;
      plans[2 * j + 1] = p.chunk;
    }
  }
  return B200RNN_OK;
}

/* test only (not declared in the public header): the folded LayerNorm prologue's kernels as a layer runs them.
   Row r < R of x (and of dx) sits at x + s_outer * (r / inner_n) + s_inner * (r % inner_n) floats; out and dy are dense
   [R][Cc]. out != NULL: out = LayerNorm(x) * gamma + beta (tc_layernorm). dy != NULL: launch_layernorm_bwd with that
   dy, dx optional (NULL: only dgamma / dbeta), accumulate into dgamma / dbeta or overwrite them; part holds part_floats
   >= 2 * 2 * NUM_SMS * Cc floats of per-CTA partials. lengths (optional, B rows per step): rows r with
   r / B >= lengths[r % B] are padding, as in a ragged batch. */
B200RNN_API int b200rnn_debug_layernorm(const float* x, int64_t s_outer, int64_t s_inner, int inner_n, int R, int Cc,
                                        const float* gamma, const float* beta, float eps, float* out, const float* dy,
                                        float* dx, float* dgamma, float* dbeta, int accumulate, float* part,
                                        size_t part_floats, const int* lengths, int B, void* stream_) {
  if (!x || !gamma || R < 1 || inner_n < 1 || (out && !beta) || (dy && (!dgamma || !dbeta || !part)) ||
      (lengths && B < 1)) {
    set_error("debug_layernorm: bad arguments");
    return B200RNN_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const RowMap rows{s_outer, s_inner, inner_n};
  if (out) {
    const int rc = tc_layernorm(x, rows, R, Cc, gamma, beta, eps, out, st, nullptr, 0, lengths, B);
    if (rc != B200RNN_OK) return rc;
  }
  if (dy) {
    if (part_floats < layernorm_bwd_scratch_floats(Cc)) {
      set_error("debug_layernorm: part holds %zu floats, %zu needed", part_floats, layernorm_bwd_scratch_floats(Cc));
      return B200RNN_ERR_INVALID;
    }
    return launch_layernorm_bwd(x, rows, dy, R, Cc, gamma, eps, dx, rows, dgamma, dbeta, accumulate, part, st, lengths,
                                B);
  }
  return B200RNN_OK;
}

/* test only (not declared in the public header): the inter-layer dropout as a layer runs it, out[i] = in[i] *
   keep(i) / (1 - p) over n elements of Philox stream stream_id at {seed, offset}; hdr: 2 uint64 of device memory for
   the resolved RNG header. Any n and any float alignment (the float4 path and the scalar tail). */
/* debug only (not declared in the public header): bytes of dynamic shared memory of one runtime-sized recurrence
 * launch shape (anyh_smem), so that tests derive the on-chip tier bounds from the function the planner uses */
B200RNN_API size_t b200rnn_debug_anyh_smem(int G, int H, int C, int BS, int bwd, int onchip, int wbytes) {
  return anyh_smem(G, H, C, BS, bwd != 0, onchip != 0, wbytes);
}

B200RNN_API int b200rnn_debug_dropout(const float* in, float* out, size_t n, float p, uint64_t seed, uint64_t offset,
                                      uint32_t stream_id, uint64_t* hdr, void* stream_) {
  if (!in || !out || !hdr) {
    set_error("debug_dropout: null pointer");
    return B200RNN_ERR_INVALID;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream_);
  const int rc = launch_rng_setup(hdr, seed, offset, nullptr, 0, st);
  if (rc != B200RNN_OK) return rc;
  return launch_dropout(in, out, n, p, hdr, stream_id, st);
}

}  // extern "C"
