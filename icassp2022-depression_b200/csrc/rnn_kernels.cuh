// rnn_kernels.cuh — host-side launch interface of the persistent recurrence kernels (K2-K5).
#pragma once
#include "common.cuh"

namespace b200rnn {

// One launch runs ALL directions of one layer: grid = D * nslices clusters of C CTAs.
// Ragged batches (lengths != NULL, the VL instantiations): batch slot q of slice s holds row order[s*BS + q], so a
// cluster holds sequences of similar length, and it runs only as many steps as its longest one; the outputs and gate
// gradients of the steps it skips are written as zeros, like those of every step past a sequence's length.
struct RecFwdParams {
  int mode, B, T, H, D;
  int training;              // save activated gates + hn/c for backward
  const float* w_hh[2];      // per direction [G*H, H]
  const float* b_hh[2];      // per direction [G*H]  (GRU: only the n third is read; r,z are pre-folded)
  float* gates[2];           // per direction [T,B,G*H]; in: x-projection + folded biases; out: activated gates
  float* extra[2];           // per direction [T,B,H]; GRU: W_hn h + b_hn ; LSTM: c_t   (training only; Elman: none)
  float* y;                  // layer output, element (t,b,d*H+j) at t*y_st + b*y_sb + d*H + j (NULL: not written)
  long long y_st, y_sb;
  float* y_pool;             // optional [B, D*H]: sum over t of the layer output (fused pooling epilogue)
  float* h_n;                // [D,B,H] of this layer
  float* c_n;                // [D,B,H] of this layer (LSTM) or NULL
  long long* trace;          // debug: per-step phase timestamps of CTA 0 / warp 0 (NULL = off), [T][8]
  const int* lengths;        // optional [B]: valid steps per sequence (PackedSequence semantics); NULL = all T
  const int* order;          // with lengths: [B] row of each batch slot, by descending length (launch_length_order)
  // streamed x-projection (D = 1 only): the GEMM writing gates[0] may still run. The x-projection of step t is read
  // only once ready[m] >= tiles_n for the row tiles m holding rows [t*B, (t+1)*B) (TC_TILE_M rows each). NULL = the
  // gates are complete at launch.
  const int* ready;
  int tiles_n;
  int tf32;                  // single-pass TF32 contraction in the tensor-core config tc8 (B200RNN_FLAG_TF32); every
                             // other config is fp32 FFMA and ignores it
  int shell_nograd;          // the no-grad forward of b200rnn_forward_fused (nothing saved, no initial state): the GRU-256
                             // tensor-core config runs on fp16 pairs (rec_fwd_h16_kernel) unless tf32 is set
  const float* h_0;          // optional [D,B,H] initial state of this layer, caller's row order (NULL: zeros)
  const float* c_0;          // optional [D,B,H] initial cell state (LSTM; NULL: zeros)
  // LSTM with a projection (rec_fwd_proj_kernel): P = proj_size, 0 = none. Then y, h_n and h_0 are P wide (y column
  // d*P + p), w_hh is [G*H, P], and m (training) receives o * tanh(c), the operand of the dW_hr GEMM
  int P;
  const float* w_hr[2];      // per direction [P, H]
  float* m[2];               // per direction [T,B,H] (training only)
  // optional, the GRU-256 fp16-pair kernel only (D = 1): W_hh of direction 0 already split, as the weight cache holds it
  // (prep_whh_h16, h16::Gru256 cache image; 16-byte aligned). NULL: the prologue splits W_hh itself
  const void* whh16[2];
};

// Several models in one launch of the runtime-sized kernels (b200rnn_desc::models): model m's clusters follow model
// m - 1's, and each pointer of the launch's params is offset by m times its model stride here (elements; 0 = shared).
// The kernels take it beside their params, which keep the layout the fixed configs are compiled against.
struct RecModels {
  int M = 1;
  long long whh[2] = {0, 0};    // weight_hh per direction (backward: for the launcher's transposes, one per distinct one)
  long long bhh[2] = {0, 0};    // forward: bias_hh per direction
  long long wprep[2] = {0, 0};  // backward: w_prep per direction
  long long saved = 0;          // gates and extra (forward: the reserve, or the scratch without save)
  long long y = 0, dy = 0;      // y; backward: dy
  long long scr = 0;            // backward: dgates, dghn, dbias_part
  long long state = 0;          // h_0, c_0, h_n, c_n; backward: dh_n, dc_n, h_0, c_0, dh_0, dc_0
};

// A recurrence launch chosen for a shape, before anything is enqueued: `nclusters` clusters of C CTAs, of which
// `capacity` can be co-resident (cudaOccupancyMaxActiveClusters). `kernel` takes (P, int nslices) or, the runtime-sized
// kernels, (P, int nslices, RecModels).
template <typename P>
struct ClusterLaunch {
  const void* kernel;
  int C, NT, nslices, nclusters, capacity;
  size_t smem;
  // a runtime-sized kernel of rnn_anyh.cu (GRU / LSTM hidden sizes other than 128 / 256, every Elman one): it takes no
  // streamed x-projection (RecFwdParams::ready). BS batch rows per cluster; onchip: W_hh stays in shared memory (else it
  // is read from L2 every step).
  bool anyh = false;
  int BS = 0;
  bool onchip = false;
  RecModels models;  // the runtime-sized kernels: the models of the launch (nclusters counts them all)
  int ctas() const { return nclusters * C; }
  bool one_wave() const { return nclusters <= capacity; }
};
using RecFwdLaunch = ClusterLaunch<RecFwdParams>;

struct RecBwdParams {
  int mode, B, T, H, D;
  const float* w_hh[2];      // per direction weight_hh [G*H, H]
  float* w_prep[2];          // per direction scratch, G*H*H floats: per-CTA transposed slices (whh_prep_kernel, filled
                             // by the launcher)
  const float* gates[2];     // saved activated gates [T,B,G*H]
  const float* extra[2];     // GRU hn / LSTM c, [T,B,H]
  const float* y;            // this layer's forward output (h_t), strided
  long long y_st, y_sb;
  const float* dy;           // gradient of this layer's output, strided (NULL: use dy_pool)
  long long dy_st, dy_sb;
  const float* dy_pool;      // [B, D*H]: gradient of the time-POOLED output, broadcast over the steps inside the kernel
  float dy_scale;            //           (x dy_scale): the [T,B,D*H] gradient of a mean / sum over time never exists
  const float* dh_n;         // [D,B,H] or NULL
  const float* dc_n;         // [D,B,H] or NULL
  float* dgates[2];          // out: [T,B,G*H] gradient w.r.t. the x-projection (dGi)
  float* dghn[2];            // out (GRU only): [T,B,H] gradient w.r.t. (W_hn h + b_hn) = dn * r
  float* dbias_part[2];      // out: [nslices][(G+1)*H] per-slice column sums (rows 0..G*H: dGi; GRU tail H: dghn);
                             //      Elman: [nslices][H], the sums of dpre
  int nslices_out;           // filled by the launcher
  const int* lengths;        // optional [B], as in the forward
  const int* order;          // with lengths: [B] row of each batch slot, as in the forward
  const float* h_0;          // the forward's initial state [D,B,H] or NULL (zeros): h_{prev} of the first step
  const float* c_0;          // the forward's initial cell state [D,B,H] or NULL (LSTM)
  float* dh_0;               // out, optional [D,B,H]: gradient w.r.t. h_0 (NULL: the last step's contraction is skipped)
  float* dc_0;               // out, optional [D,B,H]: gradient w.r.t. c_0 (LSTM)
  // LSTM with a projection (rec_bwd_proj_kernel): P = proj_size, 0 = none. Then dy, dh_n and dh_0 are P wide, w_hh is
  // read as it lies ([G*H, P]; w_prep unused), and dhp receives dh_t (dy_t plus the recurrent part), dW_hr's operand
  int P;
  const float* w_hr[2];      // per direction [P, H]
  float* dhp[2];             // out: per direction [T,B,P]
};
using RecBwdLaunch = ClusterLaunch<RecBwdParams>;

// The tangent recurrence of one layer (forward-mode AD, anyh_tangent_kernel): from the primal's saved gates, the tangent
// pre-activations and the tangent initial state, the tangent output. Launched like the runtime-sized forward (plan_anyh's
// shapes, W_hh rows staged or read from L2); M tangent directions run in one launch, clusters direction-major, each
// direction's tangent tensors at m times their stride below while every primal tensor is shared.
struct RecTanParams {
  int mode, B, T, H, D;
  const int* lengths;        // always NULL (forward mode takes no ragged batch): the slice code reads them
  const int* order;
  const float* w_hh[2];      // primal weight_hh per direction [G*H, H]
  const float* gates[2];     // the primal's saved activated gates [T,B,G*H] (Elman: h_t)
  const float* extra[2];     // ... and GRU W_hn h + b_hn / LSTM c_t [T,B,H] (Elman: NULL)
  const float* y;            // the primal layer output h_t (GRU: h_{t-1} of the next step), strided
  long long y_st, y_sb;
  const float* h_0;          // primal initial states [D,B,H] or NULL (zeros)
  const float* c_0;
  const float* pre[2];       // per direction [T,B,G*H] or NULL (0): W_ih x' + W_ih' x (+ W_hh' h_{t-1}, GRU r,z only)
  const float* preh[2];      // GRU, per direction [T,B,H] or NULL (0): W_hn' h_{t-1}
  const float* bih_dot[2];   // per direction [G*H] or NULL: tangents of bias_ih / bias_hh
  const float* bhh_dot[2];
  const float* h0_dot;       // [D,B,H] or NULL: tangents of the initial states
  const float* c0_dot;
  float* ydot;               // tangent output, element (t,b,d*H+j) at t*yd_st + b*yd_sb + d*H + j
  long long yd_st, yd_sb;
  float* hn_dot;             // [D,B,H]
  float* cn_dot;             // [D,B,H] (LSTM) or NULL
  // the stride of tangent direction m's block of each tangent tensor (elements); every primal tensor is shared
  long long m_pre, m_preh, m_bdot, m_ydot, m_state;
};
using RecTanLaunch = ClusterLaunch<RecTanParams>;

constexpr int MAX_SMEM = 232448;  // 227 KB opt-in limit per CTA on sm_90

// number of batch slices the launcher will use for this shape (needed to size dbias_part)
int rec_bwd_max_slices(int B);

// The units of CTA r of a C-CTA cluster: the H / 8 groups of 8 units split as evenly as possible, [j0, j0 + n). Every
// CTA owns at least one group when C <= H / 8; a slice of a state row is a whole number of 16-byte chunks. When C
// divides H / 8 this is the fixed configs' split, H / C units from r * H / C.
__host__ __device__ __forceinline__ void anyh_units(int H, int C, int r, int& j0, int& n) {
  const int g = H / 8, a = r * g / C, e = (r + 1) * g / C;
  j0 = 8 * a;
  n = 8 * (e - a);
}
__host__ __device__ __forceinline__ int anyh_max_units(int H, int C) { return 8 * ((H / 8 + C - 1) / C); }

// How many clusters of C CTAs of `kernel` (NT threads, smem bytes of dynamic shared memory) can be co-resident, from the
// driver; cached per (kernel, device, C, NT, smem). The first query of a kernel on a device opts it in to MAX_SMEM bytes
// and to non-portable (16-CTA) clusters; B200RNN_ERR_CUDA when that fails. A failed occupancy query is capacity 0.
int cluster_capacity(const void* kernel, int C, int NT, size_t smem, int* capacity);

// The runtime-sized recurrence (rnn_anyh.cu): the hidden sizes it takes (H % 16 == 0, 16 <= H <= 1024) and its config
// choice for the GRU / LSTM shapes the fixed configs do not cover and for every Elman shape
bool anyh_hidden_size(int H);
// bytes of dynamic shared memory of one runtime-sized launch shape: G gate blocks, C-CTA clusters of BS batch rows,
// backward or forward, weight_hh on chip (onchip) in wbytes per weight (4: fp32, 2: 16-bit)
size_t anyh_smem(int G, int H, int C, int BS, bool bwd, bool onchip, int wbytes);
// w16: the storage of weight_hh, 0 (fp32) or DT_F16 / DT_BF16 (h16.cuh): the 16-bit kernels stage half the bytes
// models: M > 1 runs M models in one launch
int plan_anyh_fwd(const RecFwdParams& p, RecFwdLaunch* out, int w16 = 0, int models = 1);
int plan_anyh_bwd(const RecBwdParams& p, RecBwdLaunch* out, int w16 = 0, int models = 1);

// forward: choose the config for p's shape (mode, H, P, B, D, lengths or not), then launch it; p.ready != NULL launches
// it with programmatic stream serialization, so that it may start while the GEMM before it still runs
// w16: the storage of p.w_hh (see plan_anyh_fwd), taken by the runtime-sized kernels; the fixed configs read fp32
// models > 1: that many models in one launch of the runtime-sized kernels (the caller fills out->models' strides)
int plan_rec_fwd(const RecFwdParams& p, RecFwdLaunch* out, int w16 = 0, int models = 1);
int launch_rec_fwd(const RecFwdLaunch& L, const RecFwdParams& p, cudaStream_t stream);
// W_hh [3*256][256] of a GRU-256 layer (16-byte aligned) -> h16::Gru256::CACHE_BYTES at img (256-byte aligned): the
// fp16 pairs and row scales the prologue of rec_fwd_h16_kernel would make, in its shared-memory order per CTA rank
int prep_whh_h16(const float* w_hh, void* img, cudaStream_t stream);
// backward: the same choice (plan_rec_bwd), then one launch that also prepares W_hh for the unprojected kernels and sets
// p.nslices_out
// whh16 (optional, with w16 != 0): per direction the 16-bit weight_hh; when the runtime-sized kernels run, W_hh is
// transposed from it in 16 bits and staged as such (p.w_prep then holds 16-bit data); otherwise p.w_hh (fp32) is used
// models (optional): several models in one launch, as in plan_rec_fwd
int plan_rec_bwd(const RecBwdParams& p, RecBwdLaunch* out, int w16 = 0, int models = 1);
int launch_rec_bwd(RecBwdParams& p, cudaStream_t stream, int w16 = 0, const void* const* whh16 = nullptr,
                   const RecModels* models = nullptr);
// the tangent recurrence (rnn_anyh.cu) at every hidden size anyh_hidden_size takes, for `directions` tangent directions
// in one launch: plan, then launch
int plan_anyh_tangent(const RecTanParams& p, RecTanLaunch* out, int directions);
int launch_rec_tangent(const RecTanParams& p, int directions, cudaStream_t stream);

}  // namespace b200rnn
