"""Do the numerics tests bite? Build the library with one small arithmetic mutation at a time and run the tests on it.

Each mutation is one textual edit of csrc/ that changes arithmetic only or removes a data store - never a barrier, a
flag or a counter, and an index only where no test it runs can then reach outside its allocation (the strided-layout
mutations, each with its reason), so that no mutated build can fault or hang - and is applied to a copy of the sources; that
copy is built (make, as build() does, reusing the tree's objects so that only the mutated file recompiles) and loaded with B200RNN_LIB. Each mutation names the new tests that must catch it and the
existing tests it is also run against. Against each build the script runs the new tests (stopping after a few
failures) and then the existing files in order, each until its first failure, stopping at the first file that fails;
it records per mutation which tests fail. A mutation that no new test catches is a hole in the suite.

    python tools/numerics_mutants.py [--only NAME ...] [--out tools/numerics_mutants_results.json]
    # build where nvcc is, run where the GPU is (the builds are kept under --build-dir and reused):
    python tools/numerics_mutants.py --build-only --build-dir build/mutants
    python tools/numerics_mutants.py --build-dir build/mutants
"""
import argparse
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "icassp2022-depression_b200")
sys.path[:0] = [ROOT, PKG]

REC_NEW = ["tests/test_gpu_numerics_f64.py"]
REC_EXISTING = ["tests/test_gpu_parity.py", "tests/test_gpu_property.py", "tests/test_gpu_coverage.py",
                "tests/test_gpu_varlen.py", "tests/test_gpu_proj.py", "tests/test_gpu_h16_fwd.py"]
GEMM_NEW = ["tests/test_gpu_grad_gemm_f64.py"]
GEMM_EXISTING = ["tests/test_gpu_gemm.py", "tests/test_gpu_gemm_f32a.py", "tests/test_gpu_grad_paths.py",
                 "tests/test_gpu_parity.py", "tests/test_gpu_tf32_mode.py"]
SHELL_NEW = ["tests/test_gpu_shell_f64.py"]
SHELL_EXISTING = ["tests/test_gpu_head.py", "tests/test_gpu_train_step.py", "tests/test_gpu_fuse_parity.py",
                  "tests/test_gpu_models.py"]
H16_NEW = ["tests/test_gpu_h16_numerics_f64.py"]
H16_EXISTING = ["tests/test_gpu_h16_modules.py"]

ANYH_NEW = ["tests/test_gpu_anyh_numerics_f64.py", "tests/test_gpu_poisoned_buffers.py"]
ANYH_EXISTING = ["tests/test_gpu_any_hidden.py", "tests/test_gpu_elman.py", "tests/test_gpu_varlen_sorted.py"]
CELL_NEW = ["tests/test_gpu_anyh_numerics_f64.py::test_cell_backward_off_default_init_vs_f64"]
CELL_EXISTING = ["tests/test_gpu_cells.py", "tests/test_gpu_elman.py"]
# caller-laid-out sequence tensors. These mutations change which element an access reaches, never whether it is a
# vector or a scalar access. Each note says why the mutated access stays inside the caller's allocation for every test
# in its lists (five of them inside the span of any view, whatever holds it), not only for the tests a run with
# --new-maxfail happens to reach
STRIDED_NEW = ["tests/test_gpu_strided_io.py"]
# forward-mode AD: the tangent GEMMs (api.cu b200rnn_forward_tangent), anyh_tangent_kernel and the linearised cells
JVP_NEW = ["tests/test_gpu_jvp_numerics_f64.py"]
JVP_EXISTING = ["tests/test_gpu_jvp.py"]
# stacked calls: what only layers l > 0 run (api.cu forward and backward layer loops)
STACK_NEW = ["tests/test_gpu_stacked_f64.py"]
STACK_EXISTING = ["tests/test_gpu_parity.py", "tests/test_gpu_proj.py", "tests/test_gpu_any_hidden.py",
                  "tests/test_gpu_elman.py", "tests/test_gpu_initial_state.py", "tests/test_gpu_shell_f64.py",
                  "tests/test_gpu_h16_modules.py"]
# tf32(v): v with its 13 low mantissa bits cleared, the operand precision of a single-pass TF32 product
_TF32 = "__uint_as_float(__float_as_uint({}) & 0xffffe000u)"

# name -> (file under csrc/, text, replacement, what it breaks, new tests, existing tests[, occurrence]). Without an
# occurrence the text must occur exactly once; with one, the occurrence-th (from 0) of several is edited: the fp32 and
# the 16-bit bodies of rnn_anyh.cu share their text, and the fp32 kernels come first in the file.
MUTATIONS = {
    "x3_drop_ah_bl": ("rnn_rec.cu", "            ptx::mma_tf32_m16n8k8(d[g][0], ah, bl);\n", "",
                      "3xTF32 tc8 recurrence: the hi(W) * lo(h) correction mma is lost", REC_NEW, REC_EXISTING),
    "f16_drop_ah_bl": ("rnn_rec.cu", "            ptx::mma_f16_m16n8k16(d[g][0], ah, bl);\n", "",
                       "fp16-pair tc8 recurrence: the hi(W) * lo(h) correction mma is lost", REC_NEW, REC_EXISTING),
    "fwdcell_drop_bhn": ("rnn_rec.cu", "const float hn = pre[2] + bhn;", "const float hn = pre[2];",
                         "every GRU forward config: b_hn left out of the candidate gate", REC_NEW, REC_EXISTING),
    "bwd_drop_one_minus_r": ("rnn_rec.cu", "const float dr = dn * hn * r * (1.f - r);", "const float dr = dn * hn * r;",
                             "GRU BPTT: the sigmoid derivative of r loses its (1 - r) factor", REC_NEW, REC_EXISTING),
    # the first MMA of a k-step zeroes the accumulator at k = 0: the one that follows takes over that flag
    "tc_drop_alo_bhi": ("gemm_tc.cu",
                        "          wgmma_tf32_m64n128k8(acc, a_lo + adv, b_hi + adv, k != 0);\n"
                        "          wgmma_tf32_m64n128k8(acc, a_hi + adv, b_lo + adv, 1);\n",
                        "          wgmma_tf32_m64n128k8(acc, a_hi + adv, b_lo + adv, k != 0);\n",
                        "presplit / MN-major tensor-core GEMM (gradient GEMMs): the lo(A) * hi(B) product is lost",
                        GEMM_NEW, GEMM_EXISTING),
    "tc_ra_drop_ah_bl": ("gemm_tc.cu",
                         "          wgmma_tf32_m64n128k8_ra(acc, &fa[8 * k + 4], b_hi + adv, k != 0);\n"
                         "          wgmma_tf32_m64n128k8_ra(acc, &fa[8 * k], b_lo + adv, 1);\n",
                         "          wgmma_tf32_m64n128k8_ra(acc, &fa[8 * k + 4], b_hi + adv, k != 0);\n",
                         "fp32-A tensor-core GEMM (forward input projection): the hi(A) * lo(W) product is lost",
                         GEMM_NEW, GEMM_EXISTING),
    "tc_epilogue_drop_accumulate": ("gemm_tc.cu", "              o.x += old.x; o.y += old.y;\n", "",
                                    "tensor-core epilogue: accumulate = 1 overwrites C instead of adding to it",
                                    GEMM_NEW, GEMM_EXISTING),
    "splitk_reduce_drop_accumulate": ("gemm_f32.cu", "    if (accumulate) s += *dst;\n", "",
                                      "split-K reduce (both paths): accumulate = 1 overwrites C", GEMM_NEW,
                                      GEMM_EXISTING),
    "ffma_epilogue_drop_accumulate": ("gemm_f32.cu", "            if (p.accumulate) o += dst[e];\n", "",
                                      "FFMA epilogue: accumulate = 1 overwrites C", GEMM_NEW, GEMM_EXISTING),
    # the three mask mutants: forward and backward (or fused and unfused) make the same mistake
    "head_keep_word_shift": ("fuse_head.cu", "  return rr[idx & 3] >= thr ? scale : 0.f;",
                             "  return rr[(idx + 1) & 3] >= thr ? scale : 0.f;",
                             "fuse head dropout: every element reads the next Philox word", SHELL_NEW, SHELL_EXISTING),
    "dropout_f4_y_word": ("misc_kernels.cu", "      v.y = rr[1] >= thr ? v.y * scale : 0.f;",
                          "      v.y = rr[2] >= thr ? v.y * scale : 0.f;",
                          "inter-layer dropout, float4 path: element 1 of a quad reads word 2", SHELL_NEW,
                          SHELL_EXISTING),
    "head_audio_out_stream": ("fuse_head.cu", ": keep_scale(seed, offset, 3, (size_t)b * Ha + (j - Ht), thr, scale);",
                              ": keep_scale(seed, offset, 2, (size_t)b * Ha + (j - Ht), thr, scale);",
                              "fuse head: the audio output dropout reuses the input stream 2", SHELL_NEW,
                              SHELL_EXISTING),
    "mlp_out_stream": ("head_kernels.cu", "if (drop) v *= keep_scale(hdr, stream_id + 1,",
                       "if (drop) v *= keep_scale(hdr, stream_id,",
                       "mlp_dropout: the output dropout reuses the input stream", SHELL_NEW, SHELL_EXISTING),
    "att_bwd_drop_tanh_deriv": ("head_kernels.cu", "const float dh = score[t] * dcj + ds[t] * q * (1.f - th * th);",
                                "const float dh = score[t] * dcj + ds[t] * q;",
                                "attention backward: d tanh loses its (1 - th^2)", SHELL_NEW, SHELL_EXISTING),
    "sce_dz_p_times_g": ("head_kernels.cu", "dz[(size_t)row * C + lane] = p * (g - dot);",
                         "dz[(size_t)row * C + lane] = p * g;",
                         "softmax_ce: dz drops the softmax Jacobian's rank-one term", SHELL_NEW, SHELL_EXISTING),
    "smoothl1_no_clamp": ("fuse_head.cu", "dt[0] = fminf(fmaxf(d, -1.f), 1.f) * invB;", "dt[0] = d * invB;",
                          "fuse head SmoothL1: the text head's gradient loses its clamp", SHELL_NEW, SHELL_EXISTING),
    "regression_no_gate": ("fuse_head.cu", "po = fmaf(gt * v, a.W[j], po);", "po = fmaf(v, a.W[j], po);",
                           "fuse head regression output: the sigmoid(modal_attn x) gate is dropped", SHELL_NEW,
                           SHELL_EXISTING),
    "ln_fwd_drop_eps": ("gemm_tc.cu",
                        "    const float rstd = rsqrtf(v / (float)Cc + eps);\n#pragma unroll\n    for (int i = 0; i < NV; ++i) {\n"
                        "      const int k = i * 128 + lane * 4;\n",
                        "    const float rstd = rsqrtf(v / (float)Cc);\n#pragma unroll\n    for (int i = 0; i < NV; ++i) {\n"
                        "      const int k = i * 128 + lane * 4;\n",
                        "LayerNorm forward: eps is left out of rstd", SHELL_NEW, SHELL_EXISTING),
    "ln_bwd_drop_xhat_mgx": ("gemm_tc.cu", "o4.y = rstd * (dv[i].y - mg - xv[i].y * mgx);", "o4.y = rstd * (dv[i].y - mg);",
                             "LayerNorm backward: one component of dx loses - xhat mean(g xhat)", SHELL_NEW,
                             SHELL_EXISTING),
    "adamw_no_decay": ("misc_kernels.cuh", "  p = p * c.decay - c.step_size", "  p = p - c.step_size",
                       "AdamW: the decoupled weight decay is lost", SHELL_NEW, SHELL_EXISTING),
    "adam_pow_bias_correction": ("misc_kernels.cuh", "  return -expm1f(t * log1pf(-(1.f - beta)));",
                                 "  return 1.f - powf(beta, t);",
                                 "Adam: the cancelling 1 - powf(beta, t) of the previous code", SHELL_NEW,
                                 SHELL_EXISTING),
    "h16_narrow_toward_zero": ("h16.cu", "__half_as_ushort(__float2half_rn(v))", "__half_as_ushort(__float2half_rz(v))",
                               "16-bit outputs: fp16 narrowing rounds toward zero instead of to nearest", H16_NEW,
                               H16_EXISTING),
    "h16_bwd_skip_valid_rows": ("api.cu", "    } else if (l == 0 && lengths) {  // x with its padding zeroed",
                                "    } else if (l == 0 && lengths && !layer_in) {  // x with its padding zeroed",
                                "16-bit backward: dW_ih reads the caller's padded rows of x (0 * NaN)", H16_NEW,
                                H16_EXISTING),
    "h16_widen_bf16_flush_subnormals": ("h16.cu", "return dt == DT_BF16 ? __uint_as_float((uint32_t)v << 16)",
                                        "return dt == DT_BF16 ? ((v & 0x7f80u) ? __uint_as_float((uint32_t)v << 16) : 0.f)",
                                        "bf16 widening flushes subnormals to zero", H16_NEW, H16_EXISTING),
    "h16_accumulate_two_roundings": ("h16.cu", "      if (accumulate) v += widen(d[c], dt);\n",
                                     "      if (accumulate) v = widen(narrow(v, dt), dt) + widen(d[c], dt);\n",
                                     "ACCUMULATE_GRADS, row path: the gradient is rounded before it is added",
                                     H16_NEW, H16_EXISTING),
    "tcl8_drop_al_bh": ("rnn_rec.cu", "            ptx::mma_f16_m16n8k16(d[g][0], al, bh);\n", "",
                        "fp16-pair tc8 / tcl8 recurrence: the lo(W) * hi(h) correction mma is lost", REC_NEW,
                        ["tests/test_gpu_lstm_h16_fwd.py"]),
    # the fp32 runtime-sized BPTT (anyh_bwd_kernel): arithmetic edits, or the removal of a data store
    "anyh_bwd_dh_tf32": ("rnn_anyh.cu", "      dh_carry = direct + sum;\n",
                         "      dh_carry = direct + " + _TF32.format("sum") + ";\n",
                         "fp32 anyh BPTT: the recurrent contraction dh = W_hh^T dg is truncated to TF32", ANYH_NEW,
                         ANYH_EXISTING, 0),
    "anyh_bwd_send_bf16": ("rnn_anyh.cu", "      const float v = (MODE == B200RNN_GRU && g == 2) ? dhn : dg[g];\n",
                           "      const float v = __bfloat162float(__float2bfloat16((MODE == B200RNN_GRU && g == 2) ? dhn "
                           ": dg[g]));\n",
                           "fp32 anyh BPTT: the gate gradient sent to the cluster is rounded to bf16", ANYH_NEW,
                           ANYH_EXISTING, 0),
    "anyh_bwd_frozen_dy": ("rnn_anyh.cu", "    const float dh = frozen ? dh_carry : dh_carry + dyv;\n",
                           "    const float dh = dh_carry + dyv;\n",
                           "fp32 anyh BPTT: dy past a row's length is added into the carried gradient", ANYH_NEW,
                           ANYH_EXISTING, 0),
    "anyh_bwd_skip_tail_zero": ("rnn_anyh.cu",
                                "#pragma unroll\n        for (int g = 0; g < G; ++g) gp[g * H] = 0.f;\n"
                                "        if (MODE == B200RNN_GRU) p.dghn[dir][((size_t)t * B + row) * H + j] = 0.f;\n",
                                "        (void)gp;\n",
                                "fp32 anyh BPTT, ragged: the gate gradients of the steps [T, p.T) a cluster skipped "
                                "are not written", ANYH_NEW, ANYH_EXISTING, 0),
    "anyh_bwd_lstm_frozen_dc": ("rnn_anyh.cu",
                                "      if (!frozen) dc_carry = dc_next;  // frozen: dh and dc pass straight through\n",
                                "      dc_carry = dc_next;\n",
                                "fp32 anyh LSTM BPTT, ragged: dc is carried through a frozen step's cell backward",
                                ANYH_NEW, ANYH_EXISTING, 0),
    "anyh_bwd_gru_vl_prev": ("rnn_anyh.cu",
                             "    const bool has_prev = step < T - 1 && !(MODE == B200RNN_GRU && VL && tp >= len);\n",
                             "    const bool has_prev = step < T - 1;\n",
                             "fp32 anyh GRU BPTT, ragged reverse half: the last valid step reads the masked 0 as its "
                             "previous state instead of h_0", ANYH_NEW, ANYH_EXISTING, 0),
    "cell_bwd_gru_dh_drop8": ("cell.cu", "      direct = gru_cell_bwd(sv, sx, hp, dh, dg, dhn);\n",
                              "      direct = gru_cell_bwd(sv, sx, hp, __uint_as_float(__float_as_uint(dh) & 0xffffff00u), "
                              "dg, dhn);\n",
                              "GRUCell backward: the output gradient loses its 8 low mantissa bits", CELL_NEW,
                              CELL_EXISTING),
    "cell_bwd_elman_dh_drop8": ("cell.cu",
                                "    const float dg = elman_cell_bwd(p.gates[(size_t)b * H + j], dh, relu);\n",
                                "    const float dg = elman_cell_bwd(p.gates[(size_t)b * H + j], "
                                "__uint_as_float(__float_as_uint(dh) & 0xffffff00u), relu);\n",
                                "RNNCell backward: the output gradient loses its 8 low mantissa bits", CELL_NEW,
                                CELL_EXISTING[1:]),
    # make_a16_map has the same line first. In bounds: the outer stride only ever gets smaller, so every box starts
    # inside the view's footprint
    "a_f32_map_drop_time_gap": ("gemm_tc.cu",
                                "  const long long si = rows.s_inner, so = dense ? (long long)M * rows.s_inner : "
                                "rows.s_outer;\n",
                                "  const long long si = rows.s_inner, so = dense ? (long long)M * rows.s_inner : "
                                "(rows.s_outer < ni * rows.s_inner ? rows.s_outer : ni * rows.s_inner);\n",
                                "fp32 input projection read in place: the 3-D map's outer (time) stride ignores a gap "
                                "between steps", STRIDED_NEW, ["tests/test_gpu_gemm_f32a.py", "tests/test_gpu_parity.py"],
                                1),
    # dense_vec's s_outer == inner_n * C term loosened to >=, on the widening's source: a time gap is taken for dense.
    # In bounds for any view without overlapping rows: the vector path reads R * C elements from its base, and such a
    # view spans at least that many
    "widen16_src_outer_ignored": ("h16.cu",
                                  "  const bool vec = dense_vec(rows, simple_rows(C), R, C, src, dst, nullptr);\n",
                                  "  const bool vec = dense_vec(rows.s_outer >= (long long)rows.inner_n * C ? "
                                  "RowMap{0, rows.s_inner, 0x7fffffff} : rows, simple_rows(C), R, C, src, dst, "
                                  "nullptr);\n",
                                  "widen16: a 16-bit x / dy with gaps between its steps is taken for dense", STRIDED_NEW,
                                  ["tests/test_gpu_h16_modules.py"]),
    # the same on the narrowing's destination: R * C elements written from the base of a y / dx that spans them
    "narrow16_dst_outer_ignored": ("h16.cu",
                                   "  const bool vec = dense_vec(dst_rows, src_rows, R, C, dst, src, wb);\n",
                                   "  const bool vec = dense_vec(dst_rows.s_outer >= (long long)dst_rows.inner_n * C ? "
                                   "RowMap{0, dst_rows.s_inner, 0x7fffffff} : dst_rows, src_rows, R, C, dst, src, "
                                   "wb);\n",
                                   "narrow16: a 16-bit y / dx with gaps between its steps is written as dense",
                                   STRIDED_NEW, ["tests/test_gpu_h16_modules.py"]),
    # The two below clamp a stride to at most its true value, so each access lands at or below the address the correct
    # code reaches in the same view: in bounds for any caller's tensor, whatever its storage.
    "rec_fwd_y_dense_rows": ("rnn_rec.cu",
                             "      if (p.y) p.y[(long long)t * p.y_st + (long long)b * p.y_sb + dir * H + j] = pend_y;\n",
                             "      if (p.y) p.y[(long long)t * p.y_st + (long long)b * (p.y_sb < p.D * H ? p.y_sb : p.D * H) "
                             "+ dir * H + j] = pend_y;\n",
                             "fixed-config forward recurrence: y's batch stride clamped to D * H (dense rows)", STRIDED_NEW,
                             ["tests/test_gpu_parity.py"]),
    "rec_bwd_dy_dense_rows": ("rnn_rec.cu",
                              "    dyv = p.dy ? p.dy[(long long)t * p.dy_st + (long long)b * p.dy_sb + dir * H + j] : "
                              "dy_pooled;\n",
                              "    dyv = p.dy ? p.dy[(long long)t * p.dy_st + (long long)b * (p.dy_sb < p.D * H ? p.dy_sb : "
                              "p.D * H) + dir * H + j] : dy_pooled;\n",
                              "fixed-config BPTT: dy's batch stride clamped to D * H (dense rows)", STRIDED_NEW,
                              ["tests/test_gpu_parity.py"]),
    # Reads the T * B * C elements from x's base, which not every tensor holds (an expanded x does not). Safe for the
    # tests it runs: the only ragged x of test_gpu_strided_io.py are compare(..., ragged=True)'s backed views, whose
    # buffers cover that dense footprint (backing), and test_gpu_varlen.py passes dense padded tensors only.
    "valid_rows_dense_src": ("misc_kernels.cu", "    dst[i] = t < lengths[b] ? src[rows.off(r) + c] : 0.f;\n",
                             "    dst[i] = t < lengths[b] ? src[(size_t)r * C + c] : 0.f;\n",
                             "ragged backward: the padding-zeroed copy of x reads row r at r * C, ignoring x's strides",
                             STRIDED_NEW, ["tests/test_gpu_varlen.py"]),
    # forward-mode AD. The stride mutations make every tangent direction read (or, in the L2 tier, also write) direction
    # 0's block of a tangent tensor: in bounds, since direction 0's block is the first of each allocation
    "jvp_gru_drop_dr_hn": ("rnn_cell.cuh", "const float dn = (1.f - n * n) * (a[2] + dr * hn + r * ahn);",
                           "const float dn = (1.f - n * n) * (a[2] + r * ahn);",
                           "GRU tangent: the candidate gate loses the dr * hn term", JVP_NEW, JVP_EXISTING),
    "jvp_lstm_drop_df_c": ("rnn_cell.cuh", "  cd = df * c_prev + fg * cd + di * gg + ig * dg;\n",
                           "  cd = fg * cd + di * gg + ig * dg;\n",
                           "LSTM tangent: the cell tangent loses df * c_prev", JVP_NEW, JVP_EXISTING),
    "jvp_drop_bhn_h_side": ("rnn_anyh.cu", "      if (MODE == B200RNN_GRU && bhh) ah += bhh[2 * H + j];\n", "",
                            "GRU tangent: b_hn' is left off the h side", JVP_NEW, JVP_EXISTING),
    "jvp_send_tf32": ("rnn_anyh.cu", "      if (s.active) h_nxt[(size_t)b * H + j] = valid ? hdn : 0.f;\n",
                      "      if (s.active) h_nxt[(size_t)b * H + j] = valid ? " + _TF32.format("hdn") + " : 0.f;\n",
                      "tangent recurrence: the tangent state sent to the cluster is rounded to TF32", JVP_NEW,
                      JVP_EXISTING),
    # the first occurrence is the backward's gradient-GEMM descriptor
    "jvp_gemm_tf32": ("api.cu", "      g.tc_tf32 = tf32 ? 1 : 0;\n", "      g.tc_tf32 = 1;\n",
                      "tangent GEMMs: single-pass TF32 whatever torch's setting", JVP_NEW, JVP_EXISTING, 1),
    "jvp_m_bdot_zero": ("api.cu", "    rp.m_bdot = GH;\n", "    rp.m_bdot = 0;\n",
                        "batched tangents: every direction reads direction 0's bias tangents", JVP_NEW, JVP_EXISTING),
    "jvp_m_preh_zero": ("api.cu", "    rp.m_pre = rp.m_preh = (long long)SS;\n",
                        "    rp.m_pre = (long long)SS;\n    rp.m_preh = 0;\n",
                        "batched tangents: every direction reads direction 0's GRU W_hn' h side", JVP_NEW, JVP_EXISTING),
    "jvp_h0_dot_direction0": ("rnn_anyh.cu",
                              "  const float* h0_dot = p.h0_dot ? p.h0_dot + m * p.m_state : nullptr;\n",
                              "  const float* h0_dot = p.h0_dot ? p.h0_dot : nullptr;\n",
                              "batched tangents: every direction starts from direction 0's h_0'", JVP_NEW, JVP_EXISTING),
    "jvp_l2_tan_ptr_direction0": ("rnn_anyh.cu",
                                  "    return base + (mdl.M > 1 ? (long long)anyh_model(p, nslices) : 0ll) * stride;\n",
                                  "    return base;\n",
                                  "batched tangents, L2 tier: every direction reads and writes direction 0's blocks",
                                  JVP_NEW, JVP_EXISTING),
    # stacked calls. The edits change a precision flag, drop a launch, pick the other of two reserve regions of the
    # same size, or overwrite instead of accumulate: every access stays where the unmutated one goes
    "stack_inner_dx_tf32": ("api.cu", '"dX"}, sl,\n                             S, tf32, st);',
                            '"dX"}, sl,\n                             S, tf32 || l > 0, st);',
                            "backward of layers l > 0: the dX GEMM (the dy of the layer below) runs single-pass TF32 "
                            "in 3xTF32 mode", STACK_NEW, STACK_EXISTING),
    "stack_inner_xproj_tf32": ("api.cu", "            g.tc_tf32 = tf32 ? 1 : 0;\n",
                               "            g.tc_tf32 = (tf32 || l > 0) ? 1 : 0;\n",
                               "forward of layers l > 0: the tensor-core x-projection runs single-pass TF32 in 3xTF32 "
                               "mode", STACK_NEW, STACK_EXISTING),
    "stack_no_inner_dropout_bwd": ("api.cu",
                                   "        rc = launch_dropout(S + sl.b_dy, S + sl.b_dy, d.TB * d.DH, d.p, hdr, "
                                   "(uint32_t)(l - 1), st);\n",
                                   "        (void)hdr;\n",
                                   "backward: the gradient through the inter-layer dropout is not masked", STACK_NEW,
                                   STACK_EXISTING),
    "stack_dw_ih_undropped": ("api.cu",
                              "X.p = layer_in ? layer_in[l - 1] : R + (drop ? rl.ydrop[l - 1] : rl.ylayer[l - 1]);",
                              "X.p = layer_in ? layer_in[l - 1] : R + rl.ylayer[l - 1];",
                              "backward: dW_ih of layer l reads layer l - 1's output before its dropout", STACK_NEW,
                              STACK_EXISTING),
    "stack_inner_dx_second_dir_overwrites": ("api.cu",
                                             "TB, Il, GH, Cx, cx_rows, k > 0, false, tc_dx, \"dX\"}",
                                             "TB, Il, GH, Cx, cx_rows, k > 0 && l == 0, false, tc_dx, \"dX\"}",
                                             "backward of layers l > 0: the reverse direction's dX overwrites the dy of "
                                             "the layer below instead of adding to it", STACK_NEW, STACK_EXISTING),
}


def gpu_info():
    q = "name,power.limit,clocks.max.sm,driver_version"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock, driver = [s.strip() for s in out.split(",")]
    except Exception as e:  # noqa: BLE001
        name, power, clock, driver = "unknown", f"unknown ({e})", "unknown", "unknown"
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock, "driver": driver}


def build(tmp, name):
    """the mutated library: copies of csrc/, the Makefile, the tree's objects and include/ under tmp, one edit, make;
    an existing build there is reused"""
    src, before, after = MUTATIONS[name][:3]
    occurrence = MUTATIONS[name][6] if len(MUTATIONS[name]) > 6 else None
    pkg = os.path.join(tmp, name, "pkg")
    lib = os.path.join(pkg, "lib", "libb200rnn.so")
    if os.path.exists(lib):
        return lib
    shutil.rmtree(os.path.join(tmp, name), ignore_errors=True)
    shutil.copytree(os.path.join(PKG, "csrc"), os.path.join(pkg, "csrc"))
    shutil.copy2(os.path.join(PKG, "Makefile"), pkg)
    if os.path.isdir(os.path.join(PKG, "build")):   # objects newer than their sources: only the edited file rebuilds
        shutil.copytree(os.path.join(PKG, "build"), os.path.join(pkg, "build"))
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, name, "include"))
    path = os.path.join(pkg, "csrc", src)
    text = open(path).read()
    if occurrence is None and text.count(before) != 1:
        raise SystemExit(f"{name}: the text to mutate occurs {text.count(before)} times in {src}")
    if occurrence is not None and text.count(before) <= occurrence:
        raise SystemExit(f"{name}: the text to mutate occurs {text.count(before)} times in {src}, not {occurrence + 1}")
    at = -1
    for _ in range((occurrence or 0) + 1):
        at = text.index(before, at + 1)
    with open(path, "w") as f:
        f.write(text[:at] + after + text[at + len(before):])
    jobs = str(max(1, min(8, os.cpu_count() or 1)))
    subprocess.run(["make", "-C", pkg, "-j", jobs], check=True, capture_output=True)
    return lib


def failing(lib, paths, maxfail=None):
    """ids of the tests in `paths` that fail (or error) against the library `lib`"""
    env = dict(os.environ, B200RNN_LIB=lib)
    cmd = [sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "-rfE", "--tb=no", *paths]
    if maxfail:
        cmd.append(f"--maxfail={maxfail}")
    out = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True).stdout
    return sorted(set(re.findall(r"^(?:FAILED|ERROR) (\S+)", out, re.M)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", nargs="*", choices=list(MUTATIONS))
    ap.add_argument("--out", default=os.path.join(ROOT, "tools", "numerics_mutants_results.json"))
    ap.add_argument("--build-dir", help="keep (and reuse) the mutated builds here instead of a temporary directory")
    ap.add_argument("--build-only", action="store_true", help="build the mutated libraries, run nothing")
    ap.add_argument("--new-maxfail", type=int, default=5, help="stop the new tests after this many failures")
    args = ap.parse_args()
    names = args.only or list(MUTATIONS)
    with tempfile.TemporaryDirectory() as tmp:
        where = os.path.abspath(args.build_dir) if args.build_dir else tmp
        if args.build_only:
            for name in names:
                print(name, build(where, name), flush=True)
            return 0
        res = {"mutations": {}}
        if os.path.exists(args.out):   # a run of some mutations (--only) adds to the results of the others
            with open(args.out) as f:
                res = json.load(f)
        res["device"] = gpu_info()
        for name in names:
            src, before, after, breaks, new_paths, old_paths = MUTATIONS[name][:6]
            lib = build(where, name)
            new = failing(lib, new_paths, maxfail=args.new_maxfail)
            old = {}
            for p in old_paths:   # the first existing file that catches the mutation is enough
                old[p] = failing(lib, [p], maxfail=1)
                if old[p]:
                    break
            res["mutations"][name] = {
                "file": src, "replaced": before.strip(), "with": after.strip(), "breaks": breaks,
                **({"occurrence": MUTATIONS[name][6]} if len(MUTATIONS[name]) > 6 else {}),
                "new_tests": new_paths, "new_tests_failing": new, "caught_by_new_tests": bool(new),
                "existing_tests_run": list(old), "existing_first_failure": {p: f[0] for p, f in old.items() if f},
                "caught_by_existing_tests": any(old.values()),
            }
            print(name, "new:", len(new), "existing:", res["mutations"][name]["caught_by_existing_tests"], flush=True)
            with open(args.out, "w") as f:   # after each mutation: a long run keeps what it has measured
                json.dump(res, f, indent=1)
                f.write("\n")
    return 0 if all(m["caught_by_new_tests"] for m in res["mutations"].values()) else 1


if __name__ == "__main__":
    sys.exit(main())
