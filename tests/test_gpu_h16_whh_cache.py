"""Frozen GRU-256 encoders keep weight_hh as fp16 pairs in the weight cache (b200rnn_prepare_weights): the no-grad fused
forward's recurrence (rec_fwd_h16_kernel) then copies its pairs and row scales instead of splitting W_hh per launch.

The cache holds exactly the pairs the uncached prologue makes, so a cached call is bitwise equal to an uncached one: fixed
length, ragged and more than one wave of clusters, through b200rnn_forward_fused and through forward_ln_sum. An in-place
edit of weight_hh refreshes the cache, and CUDA-graph replays of the cached call equal eager calls."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _gru(seed, layers=2):
    import b200rnn

    torch.manual_seed(seed)
    gru = b200rnn.GRU(256, 256, num_layers=layers).to(DEV)
    for p in gru.parameters():
        p.requires_grad_(False)
    return gru


def _fused(gru, x_tm, lengths=None, wcache=None):
    from b200rnn import _lib
    from b200rnn.functional import _make_desc, _stream_ptr

    lib = _lib.load()
    T, B, _ = x_tm.shape
    desc = _make_desc(gru._config(), B, T, False)
    _, sbytes = _lib.workspace_bytes(desc)
    scratch = torch.empty(sbytes, dtype=torch.uint8, device=DEV)
    y = torch.empty(T, B, 256, device=DEV)
    h_n = torch.empty(gru.num_layers, B, 256, device=DEV)
    params = _lib.ptr_array([w.data_ptr() for w in gru._flat_weights])
    lens = lengths.to(DEV, torch.int32).contiguous() if lengths is not None else None
    rc = lib.b200rnn_forward_fused(ctypes.byref(desc), x_tm.data_ptr(), x_tm.stride(0), x_tm.stride(1), params,
                                   y.data_ptr(), B * 256, 256, h_n.data_ptr(), None, None, scratch.data_ptr(), 0, 0,
                                   None, None, None, 0.0, None, lens.data_ptr() if lens is not None else None,
                                   wcache.data_ptr() if wcache is not None else None, None, _stream_ptr(DEV))
    _lib.check(rc, "b200rnn_forward_fused")
    return y, h_n


@pytest.mark.parametrize("B, ragged", [(128, False), (128, True), (160, False), (300, False), (5, False)],
                         ids=["b128", "b128_ragged", "b160", "b300", "b5"])
def test_cached_whh_pairs_are_bitwise_neutral(B, ragged):
    gru = _gru(B)
    cache = gru.frozen_weight_cache()
    assert cache is not None
    g = torch.Generator().manual_seed(B + ragged)
    x = torch.randn(120, B, 256, generator=g).to(DEV)
    lens = None
    if ragged:
        lens = torch.randint(1, 121, (B,), generator=g)
        lens[B // 3] = 120
    with torch.no_grad():
        y_u, h_u = _fused(gru, x, lens)
        y_c, h_c = _fused(gru, x, lens, cache)
    torch.cuda.synchronize()
    assert torch.equal(y_u, y_c) and torch.equal(h_u, h_c)


def test_pooled_features_weight_hh_edit_and_graph_replay():
    gru = _gru(7)
    ln = torch.nn.LayerNorm(256).to(DEV)
    x = torch.randn(120, 128, 256, device=DEV)
    with torch.no_grad():
        cached = gru.forward_ln_sum(x, ln).clone()
        assert gru.frozen_weight_cache() is not None
        y_u, _ = _fused(gru, x)
        y_c, _ = _fused(gru, x, wcache=gru.frozen_weight_cache())
        assert torch.equal(y_u, y_c)
        # an in-place edit of weight_hh refreshes the cache: the result equals a fresh module with the edited weights
        gru.weight_hh_l1.mul_(0.5)
        edited = gru.forward_ln_sum(x, ln).clone()
        fresh = _gru(7)
        fresh.load_state_dict(gru.state_dict())
        assert torch.equal(edited, fresh.forward_ln_sum(x, ln))
        assert not torch.equal(edited, cached)
        # graph capture of the cached call (the cache is built before capture)
        gru.frozen_weight_cache()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            gru.forward_ln_sum(x, ln)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static = gru.forward_ln_sum(x, ln)
        for i in range(5):
            xi = torch.randn_like(x)
            x.copy_(xi)
            graph.replay()
            eager = gru.forward_ln_sum(xi, ln)
            torch.cuda.synchronize()
            assert torch.equal(static, eager), f"replay {i}"
