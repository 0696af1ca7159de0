"""GPU: binding a network is all or nothing.  A dmnerf_set_weights call rejected for its arguments leaves the slot exactly as
it was: the CUDA-core and tensor-core forwards, the training forward and the 30 gradients of the backward through it are the
same bit for bit as before the call.  Raw C ABI on a context of its own, so that no binding cache sits in between."""
import ctypes as C

import pytest
import torch

from dmnerf_b200 import _lib
from dmnerf_b200.engine import ordered_params
from dmnerf_b200.testing import make_models

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
INS, M = 13, 1000


def _everything(lib, h, params, x, d_out):
    """What slot 0 computes on fixed inputs: the forward of every impl, the training forward and its 30 gradients."""
    st, p = None, _lib.ptr
    res = {}
    for name, impl in (("simt", _lib.IMPL_SIMT), ("umma", _lib.IMPL_UMMA), ("auto", _lib.IMPL_AUTO)):
        out = torch.empty(M, 5 + INS, device=DEV)
        _lib.check(lib.dmnerf_mlp_forward(h, 0, p(x), M, p(out), impl, st), "dmnerf_mlp_forward")
        res[name] = out
    out, acts = torch.empty(M, 5 + INS, device=DEV), torch.empty(M * lib.dmnerf_act_floats_per_sample(), device=DEV)
    _lib.check(lib.dmnerf_mlp_forward_train(h, 0, p(x), None, None, None, M, 1, p(out), p(acts), _lib.IMPL_UMMA, st),
               "dmnerf_mlp_forward_train")
    grads = [torch.empty_like(q) for q in params]
    scratch = torch.empty(lib.dmnerf_mlp_backward_scratch_floats(M), device=DEV)
    _lib.check(lib.dmnerf_mlp_backward(h, 0, p(acts), p(d_out), M, _lib.ptrs(grads), p(scratch), 1, st), "dmnerf_mlp_backward")
    _lib.check(lib.dmnerf_sync_check(h, st), "dmnerf_sync_check")
    res["train"] = out
    res.update(("grad %d" % i, g) for i, g in enumerate(grads))
    return res


def test_rejected_set_weights_leaves_the_slot_as_it_was():
    lib = _lib.load()
    net_a, net_b, _, _ = make_models(101, 202, INS, DEV)
    pa, pb = ordered_params(net_a)[0], ordered_params(net_b)[0]
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(M, 90, generator=g) * 0.5).to(DEV)
    d_out = (torch.randn(M, 5 + INS, generator=g) * 1e-3).to(DEV)
    torch.cuda.synchronize()
    h = C.c_void_p()
    _lib.check(lib.dmnerf_ctx_create(0, C.byref(h)), "dmnerf_ctx_create")
    try:
        _lib.check(lib.dmnerf_set_weights(h, 0, _lib.ptrs(pa), len(pa), INS, None), "dmnerf_set_weights")
        before = _everything(lib, h, pa, x, d_out)
        assert torch.equal(before["auto"], before["umma"])          # AUTO on a bound slot is the tensor-core network
        # network B with parameter 10 NULL: the call checks all 30 pointers before it takes any of them
        null10 = _lib.ptrs(pb)
        null10[10] = None
        assert lib.dmnerf_set_weights(h, 0, null10, len(pb), INS, None) != 0
        assert b"parameter 10 is NULL" in lib.dmnerf_last_error()
        for n_params, ins_num in ((len(pb) - 1, INS), (len(pb), 0), (len(pb), 128)):
            assert lib.dmnerf_set_weights(h, 0, _lib.ptrs(pb), n_params, ins_num, None) != 0, (n_params, ins_num)
        after = _everything(lib, h, pa, x, d_out)
        for k in before:
            assert torch.equal(before[k], after[k]), k
        # and B bound for real changes every forward
        _lib.check(lib.dmnerf_set_weights(h, 0, _lib.ptrs(pb), len(pb), INS, None), "dmnerf_set_weights")
        rebound = _everything(lib, h, pb, x, d_out)
        for k in ("simt", "umma", "train"):
            assert not torch.equal(before[k], rebound[k]), k
    finally:
        _lib.check(lib.dmnerf_ctx_destroy(h), "dmnerf_ctx_destroy")
