"""Drop-in ``nn.Module`` mirrors of ``torch.nn.GRU`` / ``torch.nn.LSTM`` / ``torch.nn.RNN`` backed by the sm_90a kernels.

They keep the constructor signature, parameter names / shapes / registration order
(``weight_ih_l{k}[_reverse]``, ``weight_hh_...``, ``bias_ih_...``, ``bias_hh_...``; torch rnn.py:171-216), the
default init U(-1/sqrt(H), 1/sqrt(H)) (rnn.py:308-311) and the ``forward`` return structure, so that

* ``state_dict`` round-trips with stock modules (fuse_net_whole.py:569-588 copies these keys by name),
* ``torch.save(model)`` pickles (audio_gru_whole.py:123-126),
* the reference model classes (audio_gru_whole.py:59-60, text_bilstm_whole.py:54-56,
  fuse_net_whole.py:266-268, 281-286) construct them unchanged once :func:`install` has rebound
  ``torch.nn.GRU`` / ``torch.nn.LSTM``.

``PackedSequence`` input is supported (per-sequence lengths in the kernels), and so are an initial state ``hx``
(checked as torch checks it, differentiable: streaming inference or truncated BPTT that chains ``h_n`` into the next
call) and unbatched 2-D input. ``hidden_size`` is any multiple of 16 from 16 to 1024: 128 and 256 run the tuned
fixed-size kernels, every other size the runtime-sized cluster kernels (csrc/rnn_anyh.cu); other sizes raise
``B200RNNError`` at the first forward. ``LSTM(..., proj_size=P)`` (LSTMP: ``h_t = W_hr (o_t * tanh c_t)``) runs on its own
projected kernels for P in {H/4, H/2} and registers ``weight_hr_l{k}[_reverse]`` last, as torch does. Features that
raise ``NotImplementedError``: bias=False, and other projection sizes.

``dtype=torch.float16`` / ``torch.bfloat16`` (or ``.half()``, ``.bfloat16()``, ``.to(dtype)``) gives a 16-bit module:
input, ``hx``, outputs and gradients in that dtype, the input projection on native 16-bit tensor cores, ``weight_hh``
kept 16-bit by the runtime-sized recurrence, the state carried in fp32 (DESIGN.md "16-bit modules"). It has every
feature above except ``proj_size`` and the model-shell fusions (``forward_ln_sum`` computes it unfused,
``frozen_weight_cache`` is None). A host (CPU) tensor raises ``B200RNNError`` that is also a ``NotImplementedError``: there is no CPU path.

Under ``torch.autocast("cuda")`` an fp32 module without ``proj_size`` runs as its float16 twin would, on the fp32
parameters as masters (fp32 gradients; DESIGN.md "Mixed precision"); 16-bit modules keep their dtype.

``RNN(..., nonlinearity='tanh' | 'relu')`` (the Elman network) takes the same inputs and features at every one of
those hidden sizes on the runtime-sized kernels (csrc/rnn_anyh.cu, one gate block); it has no model-shell fusion
(``forward_ln_sum`` computes it unfused, ``frozen_weight_cache`` is None) and no ``proj_size``.
"""
from __future__ import annotations

import math
import warnings
from typing import Callable, List, Optional

import torch
import torch.nn as nn

from . import _lib
from .func import check_supported
from .functional import (CellConfig, RNNConfig, cell_forward, check_forward_ad, forward_ad_active, functorch_active,
                         prepare_weights, rnn_forward, rnn_forward_fused, rnn_ln_pool_sum, tf32_enabled)

_TORCH_GRU = nn.GRU
_TORCH_LSTM = nn.LSTM
_TORCH_RNN = nn.RNN
_ELMAN_MODES = {"tanh": _lib.RNN_TANH, "relu": _lib.RNN_RELU}
# The dtype stock nn.GRU / LSTM / RNN run in under torch.autocast("cuda", dtype=...): the AutocastCUDA wrapper of
# aten::_cudnn_rnn casts the input, the states and the weights to float16 whatever the region's dtype is, bfloat16
# included (measured on the H100, pinned by tests/test_gpu_autocast.py). An fp32 module here follows it.
_AUTOCAST_DTYPE = torch.float16
_module_counter = 0


class _B200RNNBase(nn.Module):
    _mode: int = -1
    _gates: int = 0

    def __init__(self, input_size: int, hidden_size: int, num_layers: int = 1, bias: bool = True,
                 batch_first: bool = False, dropout: float = 0.0, bidirectional: bool = False,
                 proj_size: int = 0, device=None, dtype=None) -> None:
        super().__init__()
        if proj_size != 0 and self._mode != _lib.LSTM:
            raise ValueError("proj_size argument is only supported for LSTM, not RNN or GRU")
        if not bias:
            raise NotImplementedError("b200rnn: bias=False is not used by the reference and not implemented")
        if proj_size < 0:
            raise ValueError("proj_size should be a positive integer or zero to disable projections")
        if proj_size >= hidden_size > 0:
            raise ValueError("proj_size has to be smaller than hidden_size")
        if proj_size > 0 and (hidden_size not in (128, 256) or proj_size not in (hidden_size // 4, hidden_size // 2)):
            raise NotImplementedError(
                f"b200rnn: proj_size={proj_size} with hidden_size={hidden_size} is not implemented; the projected LSTM "
                "kernels take hidden_size 128 with proj_size 32 or 64, and hidden_size 256 with proj_size 64 or 128")
        if dtype not in (None, torch.float32, torch.float16, torch.bfloat16):
            raise NotImplementedError("b200rnn: the sequence modules take float32, float16 and bfloat16")
        if proj_size > 0 and dtype in (torch.float16, torch.bfloat16):
            raise NotImplementedError("b200rnn: proj_size is float32 only")
        if not isinstance(dropout, (int, float)) or not 0 <= dropout <= 1 or isinstance(dropout, bool):
            raise ValueError("dropout should be a number in range [0, 1] representing the probability of an "
                             "element being zeroed")
        if dropout > 0 and num_layers == 1:
            warnings.warn("dropout option adds dropout after all but last recurrent layer, so non-zero dropout "
                          f"expects num_layers greater than 1, but got dropout={dropout} and num_layers={num_layers}")
        if hidden_size <= 0 or num_layers <= 0:
            raise ValueError("hidden_size and num_layers must be positive")
        self.input_size = input_size
        self.hidden_size = hidden_size
        self.num_layers = num_layers
        self.bias = bias
        self.batch_first = batch_first
        self.dropout = float(dropout)
        self.bidirectional = bidirectional
        self.proj_size = int(proj_size)
        num_directions = 2 if bidirectional else 1
        gate_size = self._gates * hidden_size
        real_hidden_size = proj_size if proj_size > 0 else hidden_size

        self._flat_weights_names: List[str] = []
        for layer in range(num_layers):
            for direction in range(num_directions):
                layer_input_size = input_size if layer == 0 else real_hidden_size * num_directions
                suffix = "_reverse" if direction == 1 else ""
                shapes = ((gate_size, layer_input_size), (gate_size, real_hidden_size), (gate_size,), (gate_size,))
                names = ("weight_ih_l{}{}", "weight_hh_l{}{}", "bias_ih_l{}{}", "bias_hh_l{}{}")
                if proj_size > 0:
                    shapes += ((proj_size, hidden_size),)
                    names += ("weight_hr_l{}{}",)
                for name, shape in zip(names, shapes):
                    pname = name.format(layer, suffix)
                    self.register_parameter(
                        pname, nn.Parameter(torch.empty(shape, dtype=dtype or torch.float32, device=device)))
                    self._flat_weights_names.append(pname)
        # device-resident Philox state {seed, offset} of the inter-layer dropout; advanced by the kernels so a
        # captured CUDA graph draws a new mask per replay. Not part of the state_dict.
        global _module_counter
        _module_counter += 1
        seed = (torch.initial_seed() * 0x9E3779B97F4A7C15 + _module_counter) & 0x7FFFFFFFFFFFFFFF
        self.register_buffer("_rng_state", torch.tensor([seed, 0], dtype=torch.int64, device=device),
                             persistent=False)
        # optional hook: callable(weights) -> list of gradient target tensors (see b200rnn.dp.GradBucket)
        self._grad_sink: Optional[Callable] = None
        self._wcache = None        # (key, tensor): TF32 split of the weight_ih matrices while they are frozen
        self.reset_parameters()

    # -- torch.nn.RNNBase API surface ---------------------------------------------------------------
    def reset_parameters(self) -> None:
        stdv = 1.0 / math.sqrt(self.hidden_size) if self.hidden_size > 0 else 0
        for weight in self.parameters():
            nn.init.uniform_(weight, -stdv, stdv)

    def flatten_parameters(self) -> None:  # cuDNN-ism; parameters are used in place here
        return None

    @property
    def _flat_weights(self) -> List[torch.Tensor]:
        return [getattr(self, n) for n in self._flat_weights_names]

    @property
    def all_weights(self) -> List[List[nn.Parameter]]:
        fw = self._flat_weights
        n = 5 if self.proj_size > 0 else 4
        return [fw[i:i + n] for i in range(0, len(fw), n)]

    def extra_repr(self) -> str:
        s = "{input_size}, {hidden_size}"
        if self.proj_size != 0:
            s += ", proj_size={proj_size}"
        if self.num_layers != 1:
            s += ", num_layers={num_layers}"
        if self.batch_first is not False:
            s += ", batch_first={batch_first}"
        if self.dropout != 0:
            s += ", dropout={dropout}"
        if self.bidirectional is not False:
            s += ", bidirectional={bidirectional}"
        return s.format(**self.__dict__)

    def __setstate__(self, d):
        super().__setstate__(d)
        if "_grad_sink" not in self.__dict__:
            self._grad_sink = None
        self._wcache = None

    def __getstate__(self):
        d = self.__dict__.copy()
        d["_grad_sink"] = None  # closures over buckets are not picklable / not part of the model
        d["_wcache"] = None     # derived data
        return d

    def frozen_weight_cache(self):
        """Weight cache for the no-grad fused forward, or None: the TF32 and fp16-pair splits of every ``weight_ih``
        and, for a unidirectional GRU with hidden size 256, each layer's ``weight_hh`` as fp16 pairs in the order its
        recurrence stages them. Cached and uncached calls run the same operands and give bitwise equal results.

        None for an Elman ``RNN``, whose forward has no fused path. Only while EVERY weight of the module is frozen (``requires_grad=False``, the fuse scripts' encoders:
        fuse_net_whole.py:590-593) - nothing this library launches updates such a tensor behind PyTorch's back. The
        cache is keyed on the parameters' storage addresses and version counters, so ``load_state_dict``, ``.to()`` or
        an in-place edit refresh it; trainable modules never use it (their weights change every step anyway)."""
        if torch.compiler.is_compiling():
            return None   # keyed on storage addresses and version counters, which a traced graph does not have
        ws = self._flat_weights
        if (any(w.requires_grad for w in ws) or not ws[0].is_cuda or self.proj_size or self._gates == 1 or
                ws[0].dtype != torch.float32):
            self._wcache = None
            return None
        key = tuple((w.data_ptr(), w._version) for w in ws)
        if self._wcache is None or self._wcache[0] != key:
            if torch.cuda.is_current_stream_capturing():
                return None   # never (re)build under capture: a replay would not redo it
            self._wcache = (key, prepare_weights(ws, self._config()))
        return self._wcache[1]

    def _config(self, autocast_dtype: Optional[torch.dtype] = None) -> RNNConfig:
        """The call's configuration, built per forward call: the TF32 mode follows torch's fp32 matmul precision at
        that moment (``functional.tf32_enabled``), and the backward of the call reuses it. ``autocast_dtype``: the
        call runs in that 16-bit dtype on the fp32 parameters as masters (:meth:`_autocast_dtype`)."""
        return RNNConfig(mode=self._mode, input_size=self.input_size, hidden_size=self.hidden_size,
                         num_layers=self.num_layers, num_dirs=2 if self.bidirectional else 1,
                         dropout=self.dropout, training=self.training, batch_first=self.batch_first,
                         tf32=tf32_enabled(), proj_size=self.proj_size,
                         dtype=autocast_dtype or self._flat_weights[0].dtype, master_f32=autocast_dtype is not None)

    def _autocast_dtype(self) -> Optional[torch.dtype]:
        """The 16-bit dtype this call runs in under ``torch.autocast("cuda")``, or None (the module's own dtype). An fp32
        module without ``proj_size`` inside an enabled CUDA autocast region runs as its 16-bit twin would on its
        parameters rounded to nearest even, with the fp32 parameters as masters: their gradients come back in fp32
        (``B200RNN_FLAG_F32_PARAMS``), as through the casts of stock torch's autocast wrapper. 16-bit modules keep
        their dtype; ``proj_size`` has no 16-bit kernels and stays fp32."""
        if self.proj_size or self._flat_weights[0].dtype != torch.float32 or not torch.is_autocast_enabled("cuda"):
            return None
        return _AUTOCAST_DTYPE

    def _run_packed(self, packed, hx, cfg: RNNConfig):
        """PackedSequence path (ragged DAIC-style sequences): pad, run with per-sequence lengths, re-pack exactly like
        torch (same batch_sizes / sorted_indices; hx, h_n and c_n in the caller's original batch order: the padded
        batch is in that order already)."""
        if functorch_active():   # raised before torch's unpacking, which cannot run under torch.func either
            check_supported(cfg, packed.batch_sizes, self._grad_sink)
        if forward_ad_active(packed.data):   # stock pack_padded_sequence refuses forward AD too
            check_forward_ad(cfg, packed.batch_sizes)
        rnn_utils = nn.utils.rnn
        padded, lengths = rnn_utils.pad_packed_sequence(packed, batch_first=self.batch_first)
        out = rnn_forward(padded, self._flat_weights, cfg, self._rng_state, self._grad_sink, lengths=lengths, hx=hx)
        y = out[0]
        bdim = 0 if self.batch_first else 1
        if packed.sorted_indices is not None:
            y = y.index_select(bdim, packed.sorted_indices)
            lens_sorted = lengths.index_select(0, packed.sorted_indices.cpu())
        else:
            lens_sorted = lengths
        repacked = rnn_utils.pack_padded_sequence(y, lens_sorted, batch_first=self.batch_first, enforce_sorted=True)
        y_packed = rnn_utils.PackedSequence(repacked.data, packed.batch_sizes, packed.sorted_indices,
                                            packed.unsorted_indices)
        return (y_packed, *out[1:])

    def _hx_dims_error(self, hx, want: int) -> Optional[str]:
        """torch's message when the initial state's rank does not match the input's batchedness, else None"""
        batched = "batched 3-D" if want == 3 else "unbatched 2-D"
        if self._mode == _lib.LSTM:
            if hx[0].dim() != want or hx[1].dim() != want:
                return (f"For {batched} input, hx and cx should also be {want}-D but got ({hx[0].dim()}-D, "
                        f"{hx[1].dim()}-D) tensors")
        elif hx.dim() != want:
            return f"For {batched} input, hx should also be {want}-D but got {hx.dim()}-D tensor"
        return None

    def _run(self, input, hx):
        dt = self._autocast_dtype()
        cfg = self._config(dt)
        if dt is not None:   # autograd casts: the caller's input and states get their gradients in their own dtypes
            input = input.to(dt)
            if hx is not None:
                hx = tuple(s.to(dt) for s in hx) if isinstance(hx, (tuple, list)) else hx.to(dt)
        if isinstance(input, nn.utils.rnn.PackedSequence):
            return self._run_packed(input, hx, cfg)
        if input.dim() not in (2, 3):
            raise ValueError(f"{type(self).__name__}: Expected input to be 2D or 3D, got {input.dim()}D instead")
        batched = input.dim() == 3
        if hx is not None:
            msg = self._hx_dims_error(hx, 3 if batched else 2)
            if msg:
                raise RuntimeError(msg)
        if batched:
            return rnn_forward(input, self._flat_weights, cfg, self._rng_state, self._grad_sink, hx=hx)
        # unbatched [T, I] (and [L*D, H] states): one batch row, whatever batch_first says, as torch runs it
        batch_dim = 0 if self.batch_first else 1
        if hx is not None:
            hx = tuple(s.unsqueeze(1) for s in hx) if self._mode == _lib.LSTM else hx.unsqueeze(1)
        out = rnn_forward(input.unsqueeze(batch_dim), self._flat_weights, cfg, self._rng_state, self._grad_sink,
                          hx=hx)
        return (out[0].squeeze(batch_dim), *(s.squeeze(1) for s in out[1:]))

    def forward_ln_sum(self, input: torch.Tensor, ln: Optional[nn.LayerNorm] = None,
                       prologue_done: Optional[torch.cuda.Event] = None) -> torch.Tensor:
        """``self(ln(input))[0].sum(dim=time)`` — the audio branch of fuse_net_whole.py:360-362 / fuse_net.py:338-339.

        For a GRU / LSTM with hidden sizes 128 and 256 and the widths the tensor-core projection takes, LayerNorm is folded into the layer-0 operand preparation and the
        time sum into the last layer's step loop. Without autograd (the reference's fuse scripts run it under
        ``torch.no_grad()``, fuse_net_whole.py:337) the normalised input and the [B,T,H] output never touch HBM; under
        autograd (audio_gru_whole.py:103-108 + loss.backward()) the same fusions run in both directions
        (``b200rnn_backward_fused``: LayerNorm backward, pooled-gradient broadcast inside the BPTT kernel). Otherwise
        the same value is computed unfused.

        ``prologue_done`` (no-grad fused path): recorded on the current stream once the LayerNorm prologue is
        enqueued, before the first GEMM; on every other path, recorded before anything is enqueued.
        """
        need_grad = torch.is_grad_enabled() and (input.requires_grad or any(p.requires_grad for p in self.parameters())
                                                 or (ln is not None and any(p.requires_grad for p in ln.parameters())))
        # torch.compile / torch.export trace the unfused expression through the custom ops (b200rnn/ops.py), and so does
        # a call under torch.autocast (the fusions are fp32 only); torch.func transforms compute it through b200rnn/func.py
        # and so does forward-mode AD (a dual input or parameter)
        shape_ok = (not torch.compiler.is_compiling() and not functorch_active() and self._autocast_dtype() is None and
                    not forward_ad_active(input, *self.parameters(), *(ln.parameters() if ln is not None else ())) and
                    input.is_cuda and input.dim() == 3 and self.proj_size == 0 and
                    self._gates > 1 and self._flat_weights[0].dtype == torch.float32 and
                    self.hidden_size in (128, 256) and
                    (ln is None or (self.input_size in (128, 256, 512, 1024) and ln.elementwise_affine and
                                    ln.bias is not None)))
        fusable = not need_grad and shape_ok
        if prologue_done is not None and not fusable:
            prologue_done.record()
        if need_grad and shape_ok and not isinstance(input, nn.utils.rnn.PackedSequence):
            # training graph: LayerNorm forward+backward folded around the layer-0 GEMMs, pooled gradient broadcast
            # inside the BPTT kernel (no [T,B,H] output gradient, no LN(x) autograd tensor)
            return rnn_ln_pool_sum(input, self._flat_weights, self._config(), self._rng_state, self._grad_sink,
                                   ln.weight if ln is not None else None, ln.bias if ln is not None else None,
                                   ln.eps if ln is not None else 1e-5)
        if fusable:
            out = rnn_forward_fused(input, self._flat_weights, self._config(), self._rng_state,
                                    ln.weight if ln is not None else None, ln.bias if ln is not None else None,
                                    ln.eps if ln is not None else 1e-5, pool_sum=True,
                                    wcache=self.frozen_weight_cache(), prologue_done=prologue_done)
            return out[0]
        seq = self(ln(input) if ln is not None else input)[0]
        return seq.sum(dim=1 if self.batch_first else 0)


class GRU(_B200RNNBase):
    """``torch.nn.GRU`` (gate order r,z,n; rnn.py:1221-1224) on hand-written sm_90a kernels."""

    _mode = _lib.GRU
    _gates = 3

    def forward(self, input, hx=None):
        y, h_n = self._run(input, hx)
        return y, h_n


class LSTM(_B200RNNBase):
    """``torch.nn.LSTM`` (gate order i,f,g,o; rnn.py:842-847) on hand-written sm_90a kernels."""

    _mode = _lib.LSTM
    _gates = 4

    def forward(self, input, hx=None):
        y, h_n, c_n = self._run(input, hx)
        return y, (h_n, c_n)


class RNN(_B200RNNBase):
    """``torch.nn.RNN``, the Elman network ``h_t = tanh(W_ih x_t + b_ih + W_hh h_{t-1} + b_hh)`` (or relu), on
    hand-written sm_90a kernels. Same constructor as torch's, ``nonlinearity`` included (also as the fourth
    positional argument), with its checks and messages; the ``repr`` does not show the nonlinearity, as torch's
    does not."""

    _gates = 1

    def __init__(self, input_size: int, hidden_size: int, num_layers: int = 1, nonlinearity: str = "tanh",
                 bias: bool = True, batch_first: bool = False, dropout: float = 0.0, bidirectional: bool = False,
                 device=None, dtype=None, **kwargs) -> None:
        if "proj_size" in kwargs:
            raise ValueError("proj_size argument is only supported for LSTM, not RNN or GRU")
        if kwargs:
            raise TypeError(f"RNN.__init__() got an unexpected keyword argument '{next(iter(kwargs))}'")
        if nonlinearity not in _ELMAN_MODES:
            raise ValueError(f"Unknown nonlinearity '{nonlinearity}'. Select from 'tanh' or 'relu'.")
        self.nonlinearity = nonlinearity
        self._mode = _ELMAN_MODES[nonlinearity]
        super().__init__(input_size, hidden_size, num_layers=num_layers, bias=bias, batch_first=batch_first,
                         dropout=dropout, bidirectional=bidirectional, device=device, dtype=dtype)

    def forward(self, input, hx=None):
        y, h_n = self._run(input, hx)
        return y, h_n


class _B200CellBase(nn.Module):
    """``torch.nn.GRUCell`` / ``LSTMCell`` / ``RNNCell`` (RNNCellBase): same constructor, parameters (``weight_ih``, ``weight_hh``,
    ``bias_ih``, ``bias_hh``, registered as None with ``bias=False``), init, ``extra_repr`` and ``forward``. Any
    ``input_size`` and ``hidden_size``. One fused launch per forward (csrc/cell.cu). Not rebound by :func:`install`:
    use them by name or through :func:`from_torch`."""

    _mode: int = -1
    _gates: int = 0

    def __init__(self, input_size: int, hidden_size: int, bias: bool = True, device=None, dtype=None) -> None:
        super().__init__()
        if dtype not in (None, torch.float32):
            raise NotImplementedError("b200rnn: float32 only")
        self.input_size = input_size
        self.hidden_size = hidden_size
        self.bias = bias
        kw = dict(dtype=torch.float32, device=device)
        self.weight_ih = nn.Parameter(torch.empty((self._gates * hidden_size, input_size), **kw))
        self.weight_hh = nn.Parameter(torch.empty((self._gates * hidden_size, hidden_size), **kw))
        if bias:
            self.bias_ih = nn.Parameter(torch.empty(self._gates * hidden_size, **kw))
            self.bias_hh = nn.Parameter(torch.empty(self._gates * hidden_size, **kw))
        else:
            self.register_parameter("bias_ih", None)
            self.register_parameter("bias_hh", None)
        self.reset_parameters()

    def reset_parameters(self) -> None:
        stdv = 1.0 / math.sqrt(self.hidden_size) if self.hidden_size > 0 else 0
        for weight in self.parameters():
            nn.init.uniform_(weight, -stdv, stdv)

    def extra_repr(self) -> str:
        s = "{input_size}, {hidden_size}"
        if "bias" in self.__dict__ and self.bias is not True:
            s += ", bias={bias}"
        if "nonlinearity" in self.__dict__ and self.nonlinearity != "tanh":
            s += ", nonlinearity={nonlinearity}"
        return s.format(**self.__dict__)

    def _step(self, x: torch.Tensor, hx):
        """batched step through functional.cell_forward; the TF32 mode follows torch's setting at this call"""
        weights = [self.weight_ih, self.weight_hh] + ([self.bias_ih, self.bias_hh] if self.bias else [])
        cfg = CellConfig(mode=self._mode, input_size=self.input_size, hidden_size=self.hidden_size, bias=self.bias,
                         tf32=tf32_enabled())
        return cell_forward(x, hx, weights, cfg, type(self).__name__)


class GRUCell(_B200CellBase):
    """``torch.nn.GRUCell`` (gate order r,z,n) on the sm_90a cell kernels."""

    _mode = _lib.GRU
    _gates = 3

    def forward(self, input: torch.Tensor, hx: Optional[torch.Tensor] = None) -> torch.Tensor:
        if input.dim() not in (1, 2):
            raise ValueError(f"GRUCell: Expected input to be 1D or 2D, got {input.dim()}D instead")
        if hx is not None and hx.dim() not in (1, 2):
            raise ValueError(f"GRUCell: Expected hidden to be 1D or 2D, got {hx.dim()}D instead")
        if input.dim() == 2:
            return self._step(input, hx)
        return self._step(input.unsqueeze(0), hx.unsqueeze(0) if hx is not None else None).squeeze(0)


class LSTMCell(_B200CellBase):
    """``torch.nn.LSTMCell`` (gate order i,f,g,o) on the sm_90a cell kernels."""

    _mode = _lib.LSTM
    _gates = 4

    def forward(self, input: torch.Tensor, hx=None):
        if input.dim() not in (1, 2):
            raise ValueError(f"LSTMCell: Expected input to be 1D or 2D, got {input.dim()}D instead")
        if hx is not None:
            for idx, value in enumerate(hx):
                if value.dim() not in (1, 2):
                    raise ValueError(f"LSTMCell: Expected hx[{idx}] to be 1D or 2D, got {value.dim()}D instead")
        if input.dim() == 2:
            return self._step(input, hx)
        hx = (hx[0].unsqueeze(0), hx[1].unsqueeze(0)) if hx is not None else None
        h, c = self._step(input.unsqueeze(0), hx)
        return h.squeeze(0), c.squeeze(0)


class RNNCell(_B200CellBase):
    """``torch.nn.RNNCell`` (the Elman cell, tanh or relu) on the sm_90a cell kernels. As in torch, an unknown
    ``nonlinearity`` is accepted by the constructor and raises at ``forward``."""

    _gates = 1

    def __init__(self, input_size: int, hidden_size: int, bias: bool = True, nonlinearity: str = "tanh", device=None,
                 dtype=None) -> None:
        super().__init__(input_size, hidden_size, bias, device=device, dtype=dtype)
        self.nonlinearity = nonlinearity

    @property
    def _mode(self) -> int:
        if self.nonlinearity not in _ELMAN_MODES:
            raise RuntimeError(f"Unknown nonlinearity: {self.nonlinearity}")
        return _ELMAN_MODES[self.nonlinearity]

    def forward(self, input: torch.Tensor, hx: Optional[torch.Tensor] = None) -> torch.Tensor:
        if input.dim() not in (1, 2):
            raise ValueError(f"RNNCell: Expected input to be 1D or 2D, got {input.dim()}D instead")
        if hx is not None and hx.dim() not in (1, 2):
            raise ValueError(f"RNNCell: Expected hidden to be 1D or 2D, got {hx.dim()}D instead")
        self._mode  # noqa: B018 - the nonlinearity check, before any shape check, as torch orders them
        if input.dim() == 2:
            return self._step(input, hx)
        return self._step(input.unsqueeze(0), hx.unsqueeze(0) if hx is not None else None).squeeze(0)


def install() -> None:
    """Rebind ``torch.nn.GRU`` / ``torch.nn.LSTM`` so unmodified reference code builds the b200rnn modules. The cells
    and the Elman RNN are left alone: ``torch.nn.GRUCell`` / ``LSTMCell`` / ``RNNCell`` / ``RNN`` stay stock, so host
    code using them keeps running."""
    nn.GRU = GRU
    nn.LSTM = LSTM
    torch.nn.modules.GRU = GRU
    torch.nn.modules.LSTM = LSTM


def uninstall() -> None:
    nn.GRU = _TORCH_GRU
    nn.LSTM = _TORCH_LSTM
    torch.nn.modules.GRU = _TORCH_GRU
    torch.nn.modules.LSTM = _TORCH_LSTM


def from_torch(module: nn.Module) -> nn.Module:
    """Build the b200rnn twin of a stock ``nn.GRU`` / ``nn.LSTM`` / ``nn.RNN`` / ``nn.GRUCell`` / ``nn.LSTMCell`` /
    ``nn.RNNCell`` and copy its parameters (and nonlinearity)."""
    if isinstance(module, nn.RNNCell):
        twin = RNNCell(module.input_size, module.hidden_size, bias=module.bias, nonlinearity=module.nonlinearity)
        twin.load_state_dict(module.state_dict())
        twin.train(module.training)
        return twin
    if isinstance(module, _TORCH_RNN):
        twin = RNN(module.input_size, module.hidden_size, num_layers=module.num_layers,
                   nonlinearity=module.nonlinearity, bias=module.bias, batch_first=module.batch_first,
                   dropout=module.dropout, bidirectional=module.bidirectional)
        twin.load_state_dict(module.state_dict())
        twin.train(module.training)
        return twin
    if isinstance(module, (nn.GRUCell, nn.LSTMCell)):
        twin = (GRUCell if isinstance(module, nn.GRUCell) else LSTMCell)(module.input_size, module.hidden_size,
                                                                         bias=module.bias)
        twin.load_state_dict(module.state_dict())
        twin.train(module.training)
        return twin
    if isinstance(module, _TORCH_GRU):
        cls = GRU
    elif isinstance(module, _TORCH_LSTM):
        cls = LSTM
    else:
        raise TypeError(f"expected torch.nn.GRU, torch.nn.LSTM or torch.nn.RNN, got {type(module)}")
    twin = cls(module.input_size, module.hidden_size, num_layers=module.num_layers, bias=module.bias,
               batch_first=module.batch_first, dropout=module.dropout, bidirectional=module.bidirectional,
               proj_size=getattr(module, "proj_size", 0))
    twin.load_state_dict(module.state_dict())
    twin.train(module.training)
    return twin
