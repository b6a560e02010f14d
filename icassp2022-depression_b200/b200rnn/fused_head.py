"""Fused model-shell kernels of the fuse step (SURVEY.md §8f ranks 1 and 3), Python side.

``FusedFuseStep`` runs one fuse train step in reference semantics (fuse_net_whole.py:421-465: encoders under no_grad
with train-mode dropout, only ``fc_final.0.weight`` trainable, ``MyLoss``, Adam): the two encoder calls plus ONE
launch (``b200rnn_fuse_head``) for attention pooling, both Dropout-Linear-ReLU-Dropout heads, the model output, the
two-head loss, its weight gradient, the data-parallel gradient sum over NVLink and the Adam update. It is a drop-in
for ``pretrained_feature`` + ``forward`` + ``MyLoss`` + ``backward`` + ``optimizer.step`` of both the classification
and the regression ``fusion_net``. The single-purpose kernels (``attention_pool``, ``mlp_dropout``) stay available.
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch

from . import _lib
from .functional import _on, rnn_forward_fused
from .staging import FuseBatch


def _stream(device=None) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _require_cuda(*named) -> None:
    """Raw pointers go straight to CUDA kernels: a host tensor must fail here, loudly (no CPU path)."""
    for name, t in named:
        if t is not None and not t.is_cuda:
            raise _lib.B200RNNError(f"b200rnn: {name} is on {t.device}; the fused shell kernels run on CUDA only "
                                    "and have no CPU path")


@torch.no_grad()
def attention_pool(seq_tm: torch.Tensor, h_n: torch.Tensor, attention_layer: torch.nn.Module) -> torch.Tensor:
    """``attention_net_with_w`` on the time-major LSTM output ``seq_tm`` [T,B,2H] and ``h_n`` [L*D,B,H] -> [B,H]."""
    lib = _lib.load()
    _require_cuda(("seq", seq_tm), ("h_n", h_n), ("attention weight", attention_layer[0].weight))
    T, B, H2 = seq_tm.shape
    H = H2 // 2
    lin = attention_layer[0]
    ctx = torch.empty(B, H, dtype=torch.float32, device=seq_tm.device)
    h_n = h_n.contiguous()
    assert seq_tm.stride(2) == 1
    with _on(seq_tm.device):
        rc = lib.b200rnn_attention_pool(seq_tm.data_ptr(), seq_tm.stride(0), seq_tm.stride(1), h_n.data_ptr(),
                                        h_n.shape[0], B, T, H, lin.weight.data_ptr(), lin.bias.data_ptr(),
                                        ctx.data_ptr(), _stream(seq_tm.device))
    _lib.check(rc, "b200rnn_attention_pool")
    return ctx


class _AttentionPoolFunction(torch.autograd.Function):
    """ctx[B,H] = attention_net_with_w(seq, h_n) as ONE kernel forward and ONE kernel backward (plus the [H,B]x[B,H]
    weight-gradient product): ``b200rnn_attention_pool`` / ``b200rnn_attention_pool_bwd``."""

    @staticmethod
    def forward(ctx, seq_tm: torch.Tensor, h_n: torch.Tensor, w: torch.Tensor, b: torch.Tensor):
        lib = _lib.load()
        T, B, H2 = seq_tm.shape
        H = H2 // 2
        if seq_tm.stride(2) != 1:
            seq_tm = seq_tm.contiguous()
        h_n = h_n.contiguous()
        out = torch.empty(B, H, dtype=torch.float32, device=seq_tm.device)
        with _on(seq_tm.device):
            rc = lib.b200rnn_attention_pool(seq_tm.data_ptr(), seq_tm.stride(0), seq_tm.stride(1), h_n.data_ptr(),
                                            h_n.shape[0], B, T, H, w.data_ptr(), b.data_ptr(), out.data_ptr(),
                                            _stream(seq_tm.device))
        _lib.check(rc, "b200rnn_attention_pool")
        ctx.save_for_backward(seq_tm, h_n, w, b)
        return out

    @staticmethod
    def backward(ctx, dctx):
        from .functional import gemm

        lib = _lib.load()
        seq_tm, h_n, w, b = ctx.saved_tensors
        T, B, H2 = seq_tm.shape
        H = H2 // 2
        dev = seq_tm.device
        dctx = dctx.contiguous()
        dseq = torch.empty(T, B, H2, dtype=torch.float32, device=dev)
        dh_n = torch.empty_like(h_n)
        dqpre = torch.empty(B, H, dtype=torch.float32, device=dev)
        hsum = torch.empty(B, H, dtype=torch.float32, device=dev)
        with _on(dev):
            rc = lib.b200rnn_attention_pool_bwd(seq_tm.data_ptr(), seq_tm.stride(0), seq_tm.stride(1), h_n.data_ptr(),
                                                h_n.shape[0], B, T, H, w.data_ptr(), b.data_ptr(), dctx.data_ptr(),
                                                dseq.data_ptr(), dseq.stride(0), dseq.stride(1), dh_n.data_ptr(),
                                                dqpre.data_ptr(), hsum.data_ptr(), _stream(dev))
        _lib.check(rc, "b200rnn_attention_pool_bwd")
        dw = db = None
        if ctx.needs_input_grad[2]:     # dW[i,j] = sum_b dqpre[b,i] hsum[b,j]: A = dqpre as [K=B, M=H], B = hsum as [K=B, N=H]
            dw = gemm(dqpre, hsum, a_kcontig=False, b_kcontig=False, use_splitk=False)
        if ctx.needs_input_grad[3]:
            db = dqpre.sum(dim=0)
        return dseq, dh_n, dw, db


def attention_pool_tm(attention_layer: torch.nn.Module, seq_tm: torch.Tensor, h_n: torch.Tensor) -> torch.Tensor:
    """``attention_net_with_w`` (text_bilstm_whole.py:74-99) on the TIME-MAJOR LSTM output ``seq_tm`` [T,B,2H] and
    ``h_n`` [L*D,B,H] -> [B,H]; differentiable (one kernel each way). Falls back to the PyTorch expression only for
    shapes the kernels do not take (T*H beyond one CTA's shared memory) or non-CUDA tensors of the oracle tests."""
    lin = attention_layer[0]
    T, B, H2 = seq_tm.shape
    fits = (4 * (H2 // 2) + 2 * T + T * (H2 // 2)) * 4 <= 200 * 1024 and (2 * (H2 // 2) + T) * 4 <= 48 * 1024
    if seq_tm.is_cuda and fits and seq_tm.dtype == torch.float32:
        return _AttentionPoolFunction.apply(seq_tm, h_n, lin.weight, lin.bias)
    from .models import attention_pool as _generic

    return _generic(attention_layer, seq_tm.permute(1, 0, 2), h_n.permute(1, 0, 2))


@torch.no_grad()
def mlp_dropout(x: torch.Tensor, linear: torch.nn.Linear, p: float, training: bool, rng_hdr: Optional[torch.Tensor],
                stream_id: int) -> torch.Tensor:
    """``Dropout(p) -> linear -> ReLU -> Dropout(p)`` for a square ``linear`` (fc_out / fc_audio of fusion_net)."""
    lib = _lib.load()
    _require_cuda(("x", x), ("linear.weight", linear.weight), ("rng header", rng_hdr))
    B, n = x.shape
    assert linear.weight.shape == (n, n)
    out = torch.empty_like(x)
    with _on(x.device):
        rc = lib.b200rnn_mlp_dropout(x.data_ptr(), B, n, linear.weight.data_ptr(), linear.bias.data_ptr(),
                                     out.data_ptr(), int(training), float(p),
                                     rng_hdr.data_ptr() if rng_hdr is not None else None, stream_id, _stream(x.device))
    _lib.check(rc, "b200rnn_mlp_dropout")
    return out


class FusedFuseStep:
    """One reference-semantics fuse train step (fuse_net_whole.py:421-465 / Regression/fuse_net.py:373-412) on fused
    kernels: encoders under no_grad with train-mode dropout, only ``fc_final.0.weight`` trainable, ``MyLoss``, Adam.

    After the two encoder calls everything - attention pooling, both Dropout-Linear-ReLU-Dropout heads, the model
    output, the two-head loss, ``d fc_final.0.weight``, the data-parallel gradient sum and the Adam update - is ONE
    launch of ``b200rnn_fuse_head``. Both flavours are covered: the 2-class classification ``fusion_net`` (Softmax
    output, cross entropy) and the regression one (sigmoid ``modal_attn`` gate + ReLU output, SmoothL1, one output).

    Data parallel (``torch.distributed`` initialised, world > 1): ``exchange="peer"`` (default when CUDA IPC peer
    mapping works) sums the 3 KB gradient inside the same kernel through peer-mapped buffers over NVLink
    (:class:`b200rnn.dp.PeerComm`); ``exchange="peer_async"`` additionally defers the wait for the peers, the rank-ordered
    sum and Adam to the START of the next step on a side stream (``b200rnn_fuse_head_finish``), so a rank never idles
    for a slower one at the end of its step - same arithmetic, same update order, but ``fc_final.0.weight`` carries a
    step's update only once the next step has begun or :meth:`flush` was called; ``exchange="nccl"`` keeps the separate
    ``all_reduce`` + ``b200rnn_adamw`` launches;
    ``exchange="none"`` runs a single-replica step even when a process group exists.
    """

    def __init__(self, model, lr: float = 8e-6, betas=(0.9, 0.999), eps: float = 1e-8, bucket=None,
                 process_group=None, exchange: str = "auto", concurrent_branches: bool = True,
                 allow_fallback: bool = False):
        import torch.distributed as dist

        self.concurrent_branches = bool(concurrent_branches)
        self.split_head = bool(concurrent_branches)   # text half of the head on the text stream, before the join
        self._side = None
        self.regression = bool(getattr(model, "regression", False))
        self.C = 1 if self.regression else 2
        if model.num_classes != self.C:
            raise NotImplementedError("FusedFuseStep covers the 2-class classification fusion_net and the 1-output "
                                      f"regression fusion_net (got num_classes={model.num_classes})")
        self.model = model
        self.lr, self.betas, self.eps = float(lr), (float(betas[0]), float(betas[1])), float(eps)
        w = model.fc_final[0].weight
        _require_cuda(("model (fc_final.0.weight)", w))
        dev = w.device
        self.w = w
        self.F = model.text_hidden_dims + model.audio_hidden_dims
        n = self.C * self.F
        assert w.numel() == n and w.is_contiguous()
        self.group = process_group if process_group is not None else getattr(bucket, "group", None)
        self.world = dist.get_world_size(self.group) if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank(self.group) if self.world > 1 else 0
        self.dw = torch.zeros((n + 1 + 3) // 4 * 4, device=dev)     # gradient, then this rank's loss
        self.grad = self.dw[:n]
        self.m = torch.zeros(n, device=dev)
        self.v = torch.zeros(n, device=dev)
        self.step_count = torch.zeros((), device=dev)
        self.loss = torch.zeros((), device=dev)
        self.ticket = torch.zeros(1, dtype=torch.int32, device=dev)
        self._dw_part = None
        self.rng_hdr = torch.zeros(2, dtype=torch.int64, device=dev)
        self.rng_state = torch.tensor([(torch.initial_seed() * 2654435761 + 12345) & 0x7FFFFFFFFFFFFFFF, 0],
                                      dtype=torch.int64, device=dev)
        self.comm = None
        if exchange not in ("auto", "peer", "peer_async", "nccl", "none"):
            raise ValueError("exchange must be 'auto', 'peer', 'peer_async', 'nccl' or 'none'")
        self._aux = None
        self.comm_done = torch.zeros(1, dtype=torch.int32, device=dev)
        self.exchange = "none"
        if exchange == "none":        # single-replica step even inside an initialised process group (no collective)
            self.world, self.rank = 1, 0
        if self.world > 1:
            self.exchange = "nccl"
            if exchange in ("auto", "peer", "peer_async"):
                try:
                    from .dp import PeerComm

                    self.comm = PeerComm(dev, self.group)
                    self.exchange = "peer_async" if exchange == "peer_async" else "peer"
                except Exception:
                    if exchange in ("peer", "peer_async") and not allow_fallback:
                        raise
                # every rank must take the same path: fall back together if any rank could not map its peers
                ok = torch.tensor([1 if self.comm is not None else 0], device=dev)
                dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=self.group)
                if int(ok.item()) == 0:
                    if self.comm is not None:
                        self.comm.close()
                    self.comm, self.exchange = None, "nccl"

    def _finish_args(self) -> "_lib.FuseHeadArgs":
        m = self.model
        a = _lib.FuseHeadArgs(Ht=m.text_hidden_dims, Ha=m.audio_hidden_dims, regression=int(self.regression),
                              world=self.world, rank=self.rank, defer_exchange=1,
                              lr=self.lr, beta1=self.betas[0], beta2=self.betas[1], eps=self.eps,
                              grad_scale=1.0 / self.world, W=self.w.data_ptr(), adam_m=self.m.data_ptr(),
                              adam_v=self.v.data_ptr(), adam_step=self.step_count.data_ptr(),
                              comm_step=self.comm.step.data_ptr(), comm_done=self.comm_done.data_ptr())
        for r in range(self.world):
            a.comm_buf[r] = self.comm.bufs[r]
        return a

    @torch.no_grad()
    def flush(self) -> None:
        """``exchange="peer_async"``: apply the update of the last step (its gradient has been sent to the peers, the
        wait + sum + Adam normally run at the start of the NEXT step). Call before reading ``fc_final.0.weight`` -
        evaluation, checkpointing, the end of training. No-op in every other mode and when nothing is pending."""
        if self.exchange != "peer_async" or self.comm is None:
            return
        dev = self.w.device
        a = self._finish_args()
        with _on(dev):
            _lib.check(_lib.load().b200rnn_fuse_head_finish(ctypes.byref(a), _stream(dev)), "b200rnn_fuse_head_finish")

    def close(self) -> None:
        if self.comm is not None:
            self.flush()
            self.comm.close()
            self.comm = None

    def _text_branch(self, batch: FuseBatch):
        m = self.model
        seq, h_n, _ = rnn_forward_fused(batch.text.permute(1, 0, 2), m.lstm_net._flat_weights, m.lstm_net._config(),
                                        m.lstm_net._rng_state, wcache=m.lstm_net.frozen_weight_cache())
        return seq, h_n.contiguous()

    def _audio_branch(self, batch: FuseBatch):
        m = self.model
        return m.lstm_net_audio.forward_ln_sum(batch.audio, None if self.regression else m.ln)

    def _encoders(self, batch: FuseBatch, text_stage=None):
        """The two independent encoder branches (fuse_net_whole.py:347 text BiLSTM, :361 audio GRU). With
        ``concurrent_branches`` the audio branch - the critical path, 2 x 120 serial steps - is enqueued on a second,
        high-priority stream (fork / join by events, captured as parallel branches of the CUDA graph): its persistent
        recurrence occupies most of the 132 SMs for most of the step, the text kernels fill the rest instead of
        waiting behind it. ``text_stage(seq, h_n)`` (the text half of the head kernel) runs on the text stream before
        the join, i.e. off the critical path."""
        dev = batch.text.device
        if not self.concurrent_branches:
            seq, h_n = self._text_branch(batch)
            extra = text_stage(seq, h_n) if text_stage is not None else None
            return seq, h_n, self._audio_branch(batch), extra
        if self._side is None:
            self._side = torch.cuda.Stream(dev, priority=-1)
        main = torch.cuda.current_stream(dev)
        self._side.wait_stream(main)
        with torch.cuda.stream(self._side):
            pooled = self._audio_branch(batch)
        seq, h_n = self._text_branch(batch)
        extra = text_stage(seq, h_n) if text_stage is not None else None
        main.wait_stream(self._side)
        pooled.record_stream(main)
        return seq, h_n, pooled, extra

    def _args(self, seq, h_n, pooled, tf, af, tf_in=None) -> "_lib.FuseHeadArgs":
        """Argument block of ``b200rnn_fuse_head``. ``pooled=None``: text stage only; ``tf_in``: text stage already done."""
        m = self.model
        T, B, H2 = seq.shape
        assert seq.stride(2) == 1 and (pooled is None or pooled.is_contiguous())
        att, lt, la = m.attention_layer[0], m.fc_out[1], m.fc_audio[1]
        _require_cuda(("attention weight", att.weight), ("fc_out weight", lt.weight), ("fc_audio weight", la.weight))
        return _lib.FuseHeadArgs(
            B=B, T=T, Ht=m.text_hidden_dims, Ha=m.audio_hidden_dims, n_states=h_n.shape[0],
            training=int(m.training), p=float(m.dropout), regression=int(self.regression),
            seq_st=seq.stride(0), seq_sb=seq.stride(1), seq=seq.data_ptr() if tf_in is None else None,
            h_n=h_n.data_ptr(), tf_in=tf_in.data_ptr() if tf_in is not None else None,
            w_att=att.weight.data_ptr(), b_att=att.bias.data_ptr(), w_t=lt.weight.data_ptr(), b_t=lt.bias.data_ptr(),
            pooled=pooled.data_ptr() if pooled is not None else None, w_a=la.weight.data_ptr(), b_a=la.bias.data_ptr(),
            text_feature=tf.data_ptr() if tf_in is None else None,
            audio_feature=af.data_ptr() if af is not None else None)

    @torch.no_grad()
    def features(self, batch: FuseBatch):
        """(text_feature [B,Ht], audio_feature [B,Ha]) = ``model.pretrained_feature(batch)`` (fuse_net_whole.py:336-366)
        with the head stage of ``b200rnn_fuse_head`` only (no loss, no update)."""
        m = self.model
        lib = _lib.load()
        _require_cuda(("batch.audio", batch.audio), ("batch.text", batch.text))
        dev = batch.text.device
        seq, h_n, pooled, _ = self._encoders(batch)
        B = seq.shape[1]
        tf = torch.empty(B, m.text_hidden_dims, device=dev)
        af = torch.empty(B, m.audio_hidden_dims, device=dev)
        a = self._args(seq, h_n, pooled, tf, af)
        with _on(dev):
            if m.training and m.dropout > 0:
                consume = (B * max(m.text_hidden_dims, m.audio_hidden_dims) + 3) // 4
                _lib.check(lib.b200rnn_rng_next(self.rng_hdr.data_ptr(), self.rng_state.data_ptr(), consume,
                                                _stream(dev)), "b200rnn_rng_next")
                a.rng_state = self.rng_hdr.data_ptr()
            rc = lib.b200rnn_fuse_head(ctypes.byref(a), _stream(dev))
        _lib.check(rc, "b200rnn_fuse_head")
        return tf, af

    @torch.no_grad()
    def __call__(self, batch: FuseBatch, labels: torch.Tensor):
        """Runs the step; returns (model output [B,2] probabilities / [B,1] prediction, loss scalar tensor)."""
        lib = _lib.load()
        m = self.model
        _require_cuda(("labels", labels), ("batch.audio", batch.audio), ("batch.text", batch.text))
        dev = batch.text.device
        B = batch.text.shape[0]
        tf = torch.empty(B, m.text_hidden_dims, device=dev)
        if self.exchange == "peer_async":
            # the previous step's gradient sum + Adam, beside this step's encoders: a rank that is ahead of its peers
            # waits HERE, on a stream nothing else hangs on, instead of at the end of its head kernel
            if self._aux is None:
                self._aux = torch.cuda.Stream(dev)
            main0 = torch.cuda.current_stream(dev)
            self._aux.wait_stream(main0)
            fa = self._finish_args()
            with torch.cuda.stream(self._aux), _on(dev):
                _lib.check(lib.b200rnn_fuse_head_finish(ctypes.byref(fa), _stream(dev)), "b200rnn_fuse_head_finish")

        def text_stage(seq, h_n):
            # the text half of the head (attention pooling + fc_out) on the text branch's stream, while the audio
            # recurrence is still running; reads the same {seed, offset} the final launch will read and then advance
            a0 = self._args(seq, h_n, None, tf, None)
            a0.rng_state = self.rng_state.data_ptr()
            with _on(dev):
                _lib.check(lib.b200rnn_fuse_head(ctypes.byref(a0), _stream(dev)), "b200rnn_fuse_head (text stage)")
            return True

        seq, h_n, pooled, _ = self._encoders(batch, text_stage if self.split_head else None)
        # the kernel reads `const int64_t labels[B]` (classification) / `const float labels[B]` (regression): anything
        # else (int32 from numpy, a strided view) would be silently misread, so it is converted here; class indices
        # outside {0,1} poison the loss with NaN on the device
        want = torch.float32 if self.regression else torch.int64
        if labels.dtype != want or not labels.is_contiguous():
            labels = labels.to(want).contiguous()
        if labels.numel() != B:
            raise ValueError(f"FusedFuseStep: {labels.numel()} labels for a batch of {B}")
        af = torch.empty(B, m.audio_hidden_dims, device=dev)
        out = torch.empty(B, self.C, dtype=torch.float32, device=dev)
        need = int(lib.b200rnn_fuse_head_scratch_floats(B, m.text_hidden_dims, m.audio_hidden_dims,
                                                        int(self.regression)))
        if self._dw_part is None or self._dw_part.numel() < need:
            self._dw_part = torch.empty(need, device=dev)
        a = self._args(seq, h_n, pooled, tf, af, tf_in=tf if self.split_head else None)
        a.W = self.w.data_ptr()
        a.w_modal = m.modal_attn.weight.data_ptr() if self.regression else None
        a.labels = labels.data_ptr()
        a.out = out.data_ptr()
        a.loss = self.loss.data_ptr()
        a.dw_part = self._dw_part.data_ptr()
        a.dw = self.dw.data_ptr()
        a.ticket = self.ticket.data_ptr()
        a.rng_state = self.rng_state.data_ptr()
        a.rng_consume = (B * max(m.text_hidden_dims, m.audio_hidden_dims) + 3) // 4
        a.adam_m, a.adam_v, a.adam_step = self.m.data_ptr(), self.v.data_ptr(), self.step_count.data_ptr()
        a.lr, a.beta1, a.beta2, a.eps = self.lr, self.betas[0], self.betas[1], self.eps
        a.grad_scale = 1.0 / self.world
        a.world, a.rank = 1, 0
        a.do_adam = 1
        if self.exchange in ("peer", "peer_async"):
            a.world, a.rank = self.world, self.rank
            a.comm_step = self.comm.step.data_ptr()
            a.comm_done = self.comm_done.data_ptr()
            a.defer_exchange = 1 if self.exchange == "peer_async" else 0
            for r in range(self.world):
                a.comm_buf[r] = self.comm.bufs[r]
            if self.exchange == "peer_async":
                torch.cuda.current_stream(dev).wait_stream(self._aux)   # W must carry the previous step's update
        elif self.exchange == "nccl":
            a.do_adam = 0
        with _on(dev):
            rc = lib.b200rnn_fuse_head(ctypes.byref(a), _stream(dev))
            _lib.check(rc, "b200rnn_fuse_head")
            if self.exchange == "nccl":
                import torch.distributed as dist

                dist.all_reduce(self.grad, op=dist.ReduceOp.SUM, group=self.group)
                _lib.check(lib.b200rnn_adamw(self.w.data_ptr(), self.grad.data_ptr(), self.m.data_ptr(),
                                             self.v.data_ptr(), self.step_count.data_ptr(), self.grad.numel(), self.lr,
                                             self.betas[0], self.betas[1], self.eps, 0.0, 1.0 / self.world, 1,
                                             _stream(dev)), "b200rnn_adamw")
        return out, self.loss
