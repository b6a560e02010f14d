"""Batch-sharded data parallelism for the path (SURVEY.md §8e): one process per GPU, the model replicated,
sequences sharded over ranks, and exactly ONE all-reduce per step over a single flat fp32 gradient bucket.

The reference has no distributed code at all; this is the one parallel axis the hot path offers (independent
sequences). Gradients of every trainable parameter are views into one contiguous buffer: the wgrad GEMMs of the
b200rnn GRU/LSTM write straight into those views (``B200RNN_FLAG_ACCUMULATE_GRADS``), PyTorch's autograd accumulates
the dense shells' gradients into them in place, and ``all_reduce`` consumes the buffer as is — no pack kernel.
Backend: NCCL over NVLink / NVSwitch between the GPUs of one machine, gloo in the CPU tests.
"""
from __future__ import annotations

from typing import Iterable, List, Optional

import torch
import torch.distributed as dist

from .modules import _B200RNNBase


ALIGN_FLOATS = 64   # every view starts on a 256-byte boundary (TMA bulk copies / float4 epilogues need 16 B)


def _aligned_offsets(params: Iterable[torch.Tensor], align: int = ALIGN_FLOATS):
    """Start offsets (in floats) of per-parameter views inside one flat buffer, each rounded up to ``align``."""
    offs, off = [], 0
    for p in params:
        off = (off + align - 1) // align * align
        offs.append(off)
        off += p.numel()
    return offs, off


class GradBucket:
    """Flat gradient bucket over the trainable parameters of ``model``.

    ``p.grad`` of every trainable parameter is a view of ``flat``; the RNN wgrad kernels write into those views
    directly. The reference loops call ``optimizer.zero_grad()`` (audio_gru_whole.py:183), which since torch 2.0 sets
    ``p.grad = None``: the bucket notices dropped views and re-attaches them - RNN weights when their backward asks for
    its targets (`_sink`), dense parameters at :meth:`allreduce` (a fresh ``.grad`` is copied in once and re-bound) - so
    ``zero_grad()`` with either ``set_to_none`` value, :meth:`zero` and :meth:`zero_grad` all give the same numbers.
    """

    def __init__(self, model: torch.nn.Module, process_group: Optional[dist.ProcessGroup] = None,
                 direct_rnn_grads: bool = True):
        self.params: List[torch.nn.Parameter] = [p for p in model.parameters() if p.requires_grad]
        if not self.params:
            raise ValueError("GradBucket: the model has no trainable parameter")
        dev = self.params[0].device
        offs, total = _aligned_offsets(self.params)
        self.numel = total
        self.flat = torch.zeros(self.numel, dtype=torch.float32, device=dev)
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        self._views = {}
        self._bound: List[tuple] = []
        for p, off in zip(self.params, offs):
            v = self.flat[off:off + p.numel()].view_as(p)
            p.grad = v                            # autograd accumulates into this view in place
            self._views[p.data_ptr()] = (p, v)    # keyed by storage address: saved tensors may be re-wrapped
            self._bound.append((p, v))
        if direct_rnn_grads:
            for m in model.modules():
                if isinstance(m, _B200RNNBase):
                    m._grad_sink = self._sink

    # called from the RNN autograd function: where should the weight gradients be accumulated?
    def _sink(self, weights: Iterable[torch.Tensor]):
        out = []
        for w in weights:
            ent = self._views.get(w.data_ptr())
            if ent is None:
                out.append(None)
                continue
            p, v = ent
            if p.grad is None:                    # zero_grad(set_to_none=True) dropped the view: start from zero
                v.zero_()
                p.grad = v
            elif p.grad.data_ptr() != v.data_ptr():   # someone installed a foreign .grad: fold it in, re-bind
                v.copy_(p.grad)
                p.grad = v
            out.append(v)
        return out

    def reattach(self) -> None:
        """Bring every ``p.grad`` back into the bucket (no-op when nothing was dropped)."""
        for p, v in self._bound:
            g = p.grad
            if g is None:
                v.zero_()
                p.grad = v
            elif g.data_ptr() != v.data_ptr():
                v.copy_(g)
                p.grad = v

    @property
    def nbytes(self) -> int:
        return self.numel * 4

    @property
    def grad_scale(self) -> float:
        """1/world: what the optimiser kernel multiplies the summed gradient with (mean-reduced loss)."""
        return 1.0 / self.world

    def zero(self) -> None:
        self.reattach()
        self.flat.zero_()

    zero_grad = zero

    def allreduce(self, average: bool = True) -> None:
        """The step's single collective. ``average`` gives mean-reduced-loss semantics across shards; pass
        ``average=False`` when the optimiser kernel applies :attr:`grad_scale` itself (``b200rnn_adamw``)."""
        self.reattach()
        if self.world > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group)
            if average:
                self.flat.mul_(1.0 / self.world)


class PeerComm:
    """Peer-mapped exchange buffers for the one-shot gradient exchange fused into ``b200rnn_fuse_head``.

    NCCL's latency-bound ring costs ~100 us for the 3 KB gradient of the reference-semantics fuse step; with every
    rank's 68 KB receive buffer mapped into every process (CUDA IPC, peer access over NVLink 5 / NVSwitch) the kernel
    that produced the gradient stores it straight into its peers and polls a flag - no extra launch, no extra kernel.
    Setup only: one ``cudaMalloc`` per process and one ``all_gather`` of the 64-byte IPC handles.
    """

    def __init__(self, device, process_group: Optional[dist.ProcessGroup] = None):
        import ctypes

        from . import _lib

        if not (dist.is_available() and dist.is_initialized()):
            raise RuntimeError("PeerComm needs an initialised torch.distributed process group")
        self.group = process_group
        self.world = dist.get_world_size(process_group)
        self.rank = dist.get_rank(process_group)
        if self.world > _lib.COMM_MAX_WORLD:
            raise ValueError(f"PeerComm supports up to {_lib.COMM_MAX_WORLD} ranks (one NVSwitch domain)")
        self.device = torch.device(device)
        lib = _lib.load()
        self._lib = lib
        local = ctypes.c_void_p()
        handle = (ctypes.c_ubyte * _lib.IPC_HANDLE_BYTES)()
        with torch.cuda.device(self.device):
            _lib.check(lib.b200rnn_comm_create(ctypes.byref(local), handle), "b200rnn_comm_create")
        self.local = local.value
        mine = torch.tensor(list(handle), dtype=torch.uint8, device=self.device)
        gathered = [torch.empty_like(mine) for _ in range(self.world)]
        dist.all_gather(gathered, mine, group=process_group)
        self.bufs = [None] * self.world
        self._opened = []
        with torch.cuda.device(self.device):
            for r in range(self.world):
                if r == self.rank:
                    self.bufs[r] = self.local
                    continue
                h = (ctypes.c_ubyte * _lib.IPC_HANDLE_BYTES)(*gathered[r].cpu().tolist())
                peer = ctypes.c_void_p()
                _lib.check(lib.b200rnn_comm_open(h, ctypes.byref(peer)), "b200rnn_comm_open")
                self.bufs[r] = peer.value
                self._opened.append(peer.value)
        self.step = torch.zeros(1, dtype=torch.int32, device=self.device)   # uint32 step counter of the exchange
        dist.barrier(group=process_group)   # nobody stores into a buffer that is not mapped everywhere yet

    def close(self) -> None:
        lib = self._lib
        if lib is None:
            return
        torch.cuda.synchronize(self.device)
        if dist.is_initialized():
            dist.barrier(group=self.group)   # no peer may still be storing into (or polling) a buffer being unmapped
        with torch.cuda.device(self.device):
            for p in self._opened:
                lib.b200rnn_comm_close(p)
            lib.b200rnn_comm_destroy(self.local)
        self._opened, self.local, self._lib = [], None, None


def broadcast_parameters(model: torch.nn.Module, src: int = 0,
                         process_group: Optional[dist.ProcessGroup] = None) -> None:
    """Make every replica start from rank ``src``'s weights (one flat broadcast)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(process_group) == 1:
        return
    tensors = [p.data for p in model.parameters()] + [b.data for b in model.buffers() if b.dtype.is_floating_point]
    if not tensors:
        return
    flat = torch.cat([t.reshape(-1) for t in tensors])
    dist.broadcast(flat, src=src, group=process_group)
    off = 0
    for t in tensors:
        t.copy_(flat[off:off + t.numel()].view_as(t))
        off += t.numel()


def shard_batch(n_global: int, rank: int, world: int) -> slice:
    """Rows of the global batch owned by ``rank`` (contiguous, sizes differ by at most one)."""
    base, rem = divmod(n_global, world)
    start = rank * base + min(rank, rem)
    return slice(start, start + base + (1 if rank < rem else 0))
