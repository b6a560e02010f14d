"""Assembled train steps of the single-modality scripts (SURVEY.md §8 a7 / f3), Python side.

``train()`` of audio_gru_whole.py:161-201 / text_bilstm_whole.py:154-193 is, per batch::

    x = Variable(..., requires_grad=True); optimizer.zero_grad(); output = model(x)
    loss = criterion(output, y); loss.backward(); optimizer.step()

with ``criterion = nn.CrossEntropyLoss()`` applied to the model's *Softmax outputs* (audio_gru_whole.py:73, 308) and
``optimizer = optim.AdamW`` over two parameter groups (weight decay 1e-5, 0 for names containing 'ln'; :247-255, 307).
:class:`TrainStep` runs exactly that sequence - gradient zeroing, forward, loss, backward (dx included: the loops set
``requires_grad`` on the input), one gradient all-reduce when data parallel, AdamW - as ONE CUDA graph:

* the encoders are the b200rnn GRU / LSTM kernels (forward + BPTT), their weight gradients land directly in the flat
  gradient bucket of :class:`b200rnn.FlatAdamW`;
* Softmax + CrossEntropyLoss and its gradient are one kernel (``b200rnn_softmax_ce``) fed with the model's pre-softmax
  logits (``forward_logits``);
* the optimiser is one ``b200rnn_adamw`` launch per parameter group with the 1/world of the data-parallel mean folded in;
* the regression scripts' losses (L1 / SmoothL1 on the ReLU output, audio_bilstm_perm.py:251, text_bilstm_perm.py:247)
  are passed as a callable and stay PyTorch ops inside the same graph.
"""
from __future__ import annotations

import ctypes
from typing import Callable, Optional, Union

import torch

from . import _lib
from .functional import _on, _stream_ptr
from .optim import FlatAdamW


class _SoftmaxCE(torch.autograd.Function):
    """(probs, loss) = (softmax(z), CrossEntropyLoss(softmax(z), y)); backward is the gradient computed in the same pass."""

    @staticmethod
    def forward(ctx, z: torch.Tensor, labels: torch.Tensor):
        lib = _lib.load()
        if not z.is_cuda:
            raise _lib.B200RNNError("b200rnn: softmax_ce runs on CUDA only (no CPU path)")
        z = z.contiguous()
        B, C = z.shape
        if labels.dtype != torch.int64 or not labels.is_contiguous():
            labels = labels.to(torch.int64).contiguous()
        probs = torch.empty_like(z)
        dz = torch.empty_like(z)
        row = torch.empty(B, dtype=torch.float32, device=z.device)
        loss = torch.empty((), dtype=torch.float32, device=z.device)
        with _on(z.device):
            rc = lib.b200rnn_softmax_ce(z.data_ptr(), labels.data_ptr(), B, C, probs.data_ptr(), dz.data_ptr(),
                                        row.data_ptr(), loss.data_ptr(), _stream_ptr(z.device))
        _lib.check(rc, "b200rnn_softmax_ce")
        ctx.save_for_backward(dz)
        ctx.mark_non_differentiable(probs)
        return probs, loss

    @staticmethod
    def backward(ctx, _dprobs, dloss):
        (dz,) = ctx.saved_tensors
        return dz * dloss, None


def softmax_cross_entropy(logits: torch.Tensor, labels: torch.Tensor):
    """``p = Softmax(logits); loss = CrossEntropyLoss()(p, labels)`` as the reference computes it, fused (fwd + bwd)."""
    return _SoftmaxCE.apply(logits, labels)


class TrainStep:
    """One optimisation step of a single-modality model as a CUDA graph (see module docstring).

    ``loss``: ``"softmax_ce"`` (classification scripts; needs ``model.forward_logits``) or a callable
    ``loss(output, y) -> scalar`` applied to ``model(x)`` (regression scripts).
    ``step(x, y)`` copies the batch into the graph's static buffers, replays, and returns ``(output, loss)`` tensors
    that are overwritten by the next call.
    """

    def __init__(self, model: torch.nn.Module, optimizer: FlatAdamW, x_shape, y_shape=None,
                 loss: Union[str, Callable] = "softmax_ce", y_dtype=torch.int64, use_graph: bool = True,
                 input_requires_grad: bool = True):
        p0 = next(model.parameters())
        if not p0.is_cuda:
            raise _lib.B200RNNError("b200rnn.TrainStep: the model is not on a CUDA device - no CPU path")
        self.model, self.opt, self.loss_kind = model, optimizer, loss
        dev = p0.device
        self.device = dev
        self.x = torch.zeros(tuple(x_shape), dtype=torch.float32, device=dev)
        self.y = torch.zeros(tuple(y_shape) if y_shape is not None else (x_shape[0],), dtype=y_dtype, device=dev)
        self.input_requires_grad = input_requires_grad
        self.out: Optional[torch.Tensor] = None
        self.loss_value: Optional[torch.Tensor] = None
        self.dx: Optional[torch.Tensor] = None
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.use_graph = use_graph
        self._captured = False

    # the sequence of train() in the reference, verbatim
    def _body(self):
        self.opt.zero_grad()
        x = self.x.detach().requires_grad_(self.input_requires_grad)   # Variable(..., requires_grad=True)
        if self.loss_kind == "softmax_ce":
            out, loss = softmax_cross_entropy(self.model.forward_logits(x), self.y)
        else:
            out = self.model(x)
            loss = self.loss_kind(out, self.y)
        loss.backward()
        self.opt.allreduce()
        self.opt.step()
        return out.detach(), loss.detach(), x.grad

    def _capture(self):
        side = torch.cuda.Stream(self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):      # warm-up outside the capture: allocations, lazy kernel attributes
            for _ in range(2):
                self._body()
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out, self.loss_value, self.dx = self._body()
        self._captured = True

    def warmup_and_capture(self, state_snapshot: bool = True) -> None:
        """Capture the graph. The warm-up steps would advance the weights and the Adam state, so they run on a
        snapshot that is restored before the capture (``state_snapshot``)."""
        if not self.use_graph or self._captured:
            return
        snap = None
        if state_snapshot:
            snap = ([g.flat_p.clone() for g in self.opt.groups], [g.m.clone() for g in self.opt.groups],
                    [g.v.clone() for g in self.opt.groups], self.opt.step_count.clone())
        self._capture()
        if snap is not None:
            with torch.no_grad():
                for g, p, m, v in zip(self.opt.groups, *snap[:3]):
                    g.flat_p.copy_(p); g.m.copy_(m); g.v.copy_(v)
                self.opt.step_count.copy_(snap[3])

    def step(self, x: torch.Tensor, y: torch.Tensor):
        self.x.copy_(x, non_blocking=True)
        self.y.copy_(y, non_blocking=True)
        if self.use_graph:
            if not self._captured:
                self.warmup_and_capture()
            self.graph.replay()
        else:
            self.out, self.loss_value, self.dx = self._body()
        return self.out, self.loss_value


class FuseFineTuneStep(TrainStep):
    """The fuse step with EVERY parameter trainable (SURVEY.md §3.3 (b): the end-to-end fine-tune variant of
    fuse_net_whole.py:421-465 / the all-``requires_grad`` setting of Regression/fuse_net.py:578-583 with the encoders
    inside autograd): BiLSTM + GRU forward and BPTT, attention, both heads, ``MyLoss``, ONE all-reduce over the
    10.46 MB gradient bucket, Adam (``FlatAdamW`` with weight decay 0) - captured as one CUDA graph.
    """

    def __init__(self, model, optimizer: FlatAdamW, batch: int, t_audio: int, t_text: int, criterion=None,
                 use_graph: bool = True):
        from .models import MyLoss

        super().__init__(model, optimizer, (batch, t_audio, model.audio_embed_size), (batch,), loss="fuse",
                         y_dtype=torch.float32 if model.regression else torch.int64, use_graph=use_graph,
                         input_requires_grad=False)
        self.text = torch.zeros(batch, t_text, model.text_embed_size, dtype=torch.float32, device=self.device)
        self.criterion = criterion or MyLoss(model.text_hidden_dims, regression=model.regression)

    def _body(self):
        from .fused_head import attention_pool_tm

        m = self.model
        self.opt.zero_grad()
        seq, (h_n, _) = m.lstm_net(self.text.permute(1, 0, 2))
        tf = m.fc_out(attention_pool_tm(m.attention_layer, seq, h_n))
        af = m.fc_audio(m.lstm_net_audio.forward_ln_sum(self.x, None if m.regression else m.ln))
        out = m(torch.cat((tf, af), dim=1))
        loss = self.criterion(tf, af, self.y, m)
        loss.backward()
        self.opt.allreduce()
        self.opt.step()
        return out.detach(), loss.detach(), None

    def step(self, audio: torch.Tensor, text: torch.Tensor, y: torch.Tensor):
        self.text.copy_(text, non_blocking=True)
        return super().step(audio, y)
