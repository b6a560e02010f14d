"""Argument checks of the split classification head of ``b200rnn_fuse_head`` (``halves`` set): they run on the host,
before anything touches the device, so no GPU is needed. The pointers are never dereferenced."""
import ctypes

from b200rnn import _lib

P = 256   # a non-null stand-in for a device pointer


def _args(**kw):
    a = _lib.FuseHeadArgs(B=128, T=30, Ht=128, Ha=256, n_states=4, halves=P, W=P, dw_part=P)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _rc(a):
    return _lib.load().b200rnn_fuse_head(ctypes.byref(a), None)


def test_halves_rejects_regression_and_both_branches_in_one_launch():
    lib = _lib.load()
    for bad in (dict(regression=1, pooled=P, w_a=P, b_a=P),                     # classification only
                dict(pooled=P, w_a=P, b_a=P, tf_in=P),                          # one branch per launch
                dict(pooled=P, w_a=P, b_a=P, seq=P, h_n=P, w_att=P, b_att=P, w_t=P, b_t=P),
                dict(pooled=P, w_a=P, b_a=P, dw_part=None),                     # the feature matrix goes to dw_part
                dict(pooled=P, w_a=P, b_a=P, W=None),                           # the halves read fc_final.0.weight
                dict(pooled=P, w_a=P, b_a=P, halves=P + 4)):                    # read as float4: 16-byte aligned
        assert _rc(_args(**bad)) == -1, bad
        assert b"halves" in lib.b200rnn_last_error()


def test_halves_loss_launch_needs_the_loss_arguments():
    lib = _lib.load()
    assert _rc(_args()) == -1                    # neither branch: the loss launch, without labels / dw / loss / ticket
    assert b"loss stage needs" in lib.b200rnn_last_error()
    assert _rc(_args(labels=P, dw=P, loss=P, ticket=P, do_adam=1)) == -1
    assert b"Adam stage needs" in lib.b200rnn_last_error()
    assert _rc(_args(pooled=P, w_a=None, b_a=P)) == -1     # an audio launch without fc_audio
    assert b"null pointer" in lib.b200rnn_last_error()
