"""Flat, fused AdamW for the training loops of the reference (SURVEY.md §8f rank 3).

``audio_gru_whole.py:247-255, 307`` / ``text_bilstm_whole.py:237-245, 303`` build ``optim.AdamW`` with two parameter
groups (weight decay 1e-5, and 0 for names containing ``ln``). ``FlatAdamW`` re-homes every parameter of a group as a
view of ONE contiguous buffer, keeps ``.grad``, ``m`` and ``v`` the same way, and updates a whole group with a single
kernel launch (``b200rnn_adamw``) — the flat gradient buffer is also exactly what the data-parallel step all-reduces
(one collective per step), and the ``1/world`` averaging is folded into the update.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence

import torch
import torch.distributed as dist

from . import _lib
from .dp import _aligned_offsets
from .modules import _B200RNNBase


class _Group:
    def __init__(self, params: List[torch.nn.Parameter], weight_decay: float, flat_g: torch.Tensor):
        self.params = params
        self.weight_decay = float(weight_decay)
        dev = params[0].device
        offs, n = _aligned_offsets(params)     # 256-byte aligned views: weight_hh feeds TMA bulk copies
        assert flat_g.numel() == n
        self.flat_p = torch.zeros(n, dtype=torch.float32, device=dev)
        self.flat_g = flat_g                   # a slice of the optimiser-wide gradient bucket (ONE all-reduce per step)
        self.m = torch.zeros(n, dtype=torch.float32, device=dev)
        self.v = torch.zeros(n, dtype=torch.float32, device=dev)
        self.views = []
        with torch.no_grad():
            for p, off in zip(params, offs):
                k = p.numel()
                self.flat_p[off:off + k].copy_(p.reshape(-1))
                p.data = self.flat_p[off:off + k].view_as(p)       # parameter now lives in the flat buffer
                g = self.flat_g[off:off + k].view_as(p)
                p.grad = g                                         # autograd accumulates into the flat gradient
                self.views.append((p, g))


class FlatAdamW:
    """``torch.optim.AdamW`` semantics (decoupled weight decay, no amsgrad) over flat parameter groups.

    ``groups``: sequence of ``{"params": [...], "weight_decay": wd}`` like the reference's ``optimizer_grouped_parameters``.
    """

    def __init__(self, groups: Sequence[dict], lr: float, betas=(0.9, 0.999), eps: float = 1e-8,
                 model: Optional[torch.nn.Module] = None, process_group=None):
        self.lr, self.betas, self.eps = float(lr), (float(betas[0]), float(betas[1])), float(eps)
        plist = [([p for p in g["params"] if p.requires_grad], g.get("weight_decay", 0.0))
                 for g in groups if any(p.requires_grad for p in g["params"])]
        _lib.require_fp32_params([p for ps, _ in plist for p in ps], "FlatAdamW")
        dev = plist[0][0][0].device
        sizes = [(_aligned_offsets(ps)[1] + 63) // 64 * 64 for ps, _ in plist]
        # every group's gradients live in ONE contiguous bucket: the data-parallel step all-reduces it with a single
        # collective (SURVEY.md 8e), the per-group AdamW launches read their slice of it
        self.bucket = torch.zeros(sum(sizes), dtype=torch.float32, device=dev)
        self.groups, off = [], 0
        for (ps, wd), n_al in zip(plist, sizes):
            n = _aligned_offsets(ps)[1]
            self.groups.append(_Group(ps, wd, self.bucket[off:off + n]))
            off += n_al
        self.step_count = torch.zeros((), dtype=torch.float32, device=dev)
        self.process_group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        if model is not None:   # RNN wgrad kernels write straight into the flat gradient views
            views = {p.data_ptr(): (p, v) for g in self.groups for p, v in g.views}

            def sink(weights, _v=views):
                out = []
                for w in weights:
                    ent = _v.get(w.data_ptr())
                    if ent is None:
                        out.append(None)
                        continue
                    p, v = ent
                    if p.grad is None:            # a foreign zero_grad(set_to_none=True): restart this view from zero
                        v.zero_()
                        p.grad = v
                    out.append(v)
                return out

            for mod in model.modules():
                if isinstance(mod, _B200RNNBase):
                    mod._grad_sink = sink

    @classmethod
    def like_reference(cls, model: torch.nn.Module, lr: float, weight_decay: float = 1e-5, **kw) -> "FlatAdamW":
        """The grouping of audio_gru_whole.py:247-255: no decay for parameters whose name contains 'ln'."""
        named = list(model.named_parameters())
        decay = [p for n, p in named if "ln" not in n]
        no_decay = [p for n, p in named if "ln" in n]
        groups = [{"params": decay, "weight_decay": weight_decay}]
        if no_decay:
            groups.append({"params": no_decay, "weight_decay": 0.0})
        return cls(groups, lr, model=model, **kw)

    def reattach(self) -> None:
        """Re-bind ``p.grad`` views dropped by someone else's ``zero_grad(set_to_none=True)``; fold in fresh grads."""
        for g in self.groups:
            for p, v in g.views:
                if p.grad is None:
                    v.zero_()
                    p.grad = v
                elif p.grad.data_ptr() != v.data_ptr():
                    v.copy_(p.grad)
                    p.grad = v

    def zero_grad(self, set_to_none: bool = False) -> None:   # the views are the optimiser's own storage: never dropped
        self.reattach()
        self.bucket.zero_()

    def allreduce(self) -> None:
        """The step's single collective: one all-reduce over the bucket that holds every group's gradients (the 1/world
        of the mean is folded into the AdamW kernel)."""
        self.reattach()
        if self.world > 1:
            dist.all_reduce(self.bucket, op=dist.ReduceOp.SUM, group=self.process_group)

    @property
    def nbytes(self) -> int:
        return self.bucket.numel() * 4

    @torch.no_grad()
    def step(self) -> None:
        if not all(g.flat_p.is_cuda for g in self.groups):
            raise _lib.B200RNNError("b200rnn.FlatAdamW: parameters are not on a CUDA device - no CPU path")
        lib = _lib.load()
        self.reattach()
        dev = self.groups[0].flat_p.device
        scale = 1.0 / self.world
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            for i, g in enumerate(self.groups):
                last = i == len(self.groups) - 1
                _lib.check(lib.b200rnn_adamw(g.flat_p.data_ptr(), g.flat_g.data_ptr(), g.m.data_ptr(), g.v.data_ptr(),
                                             self.step_count.data_ptr(), g.flat_p.numel(), self.lr, self.betas[0],
                                             self.betas[1], self.eps, g.weight_decay, scale, int(last), stream),
                           "b200rnn_adamw")
