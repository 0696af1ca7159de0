"""Per-device handle on the native renderer: owns a `dmnerf_ctx`, tracks which nn.Module's parameters
are bound to the coarse / fine slot and re-binds (re-packs the tensor-core operand image) whenever a
parameter's storage or version counter changed (the optimizer updates weights in place every step,
reference train_dmsr.py:62-64)."""
import ctypes as C

import torch

from . import _lib
from .synth import param_names

_contexts = {}


def _cuda_index(device):
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("dmnerf_b200 runs on CUDA devices only (got %s); there is no CPU fallback" % device)
    return device.index if device.index is not None else torch.cuda.current_device()


def get_context(device):
    idx = _cuda_index(device)
    ctx = _contexts.get(idx)
    if ctx is None:
        ctx = _contexts[idx] = Context(idx)
    return ctx


_param_cache = {}      # id(model) -> (weakref to the model, [(owner module, leaf name, parameter)], ins_num)


def ordered_params(model):
    """The 30 parameter tensors of a DM_NeRF-shaped module in reference state_dict order.  The walk over the module tree is
    cached per model (a renderer called per 4096-ray chunk does this twice per call); the cache entry is revalidated against
    the modules' own parameter tables, so re-assigned Parameter objects are picked up."""
    import weakref
    hit = _param_cache.get(id(model))
    if hit is not None and hit[0]() is model and all(mod._parameters.get(leaf) is prm for mod, leaf, prm in hit[1]):
        return [prm for _, _, prm in hit[1]], hit[2]
    params, ins_num = _ordered_params_walk(model)
    owners = {}
    for mname, mod in model.named_modules():
        for leaf, prm in mod._parameters.items():
            if prm is not None:
                owners[id(prm)] = (mod, leaf)
    try:
        _param_cache[id(model)] = (weakref.ref(model), [owners[id(prm)] + (prm,) for prm in params], ins_num)
        if len(_param_cache) > 64:
            for k in [k for k, v in _param_cache.items() if v[0]() is None]:
                del _param_cache[k]
    except (KeyError, TypeError):
        pass
    return params, ins_num


def _ordered_params_walk(model):
    named = dict(model.named_parameters())
    ins_num = named["ins_linear.weight"].shape[0] - 1
    names = param_names(ins_num)
    missing = [n for n in names if n not in named]
    if missing:
        raise RuntimeError("model is not DM_NeRF-shaped; missing parameters: %s" % missing[:4])
    return [named[n] for n in names], ins_num


class Context:
    def __init__(self, index):
        self.index = index
        self.lib = _lib.load()
        h = C.c_void_p()
        with torch.cuda.device(index):
            torch.cuda.init()
            _lib.check(self.lib.dmnerf_ctx_create(index, C.byref(h)), "dmnerf_ctx_create")
        self.handle = h
        self._bound = [None, None]     # per slot: (id(model), ((data_ptr, version), ...))
        self._keepalive = [None, None]

    def stream(self):
        # every native call looks the stream up: take the raw handle rather than building a torch.cuda.Stream each time
        return C.c_void_p(torch._C._cuda_getCurrentRawStream(self.index))

    def bind(self, slot, model):
        params, ins_num = ordered_params(model)
        key = (id(model), tuple((p.data_ptr(), p._version) for p in params))
        if self._bound[slot] == key:
            return ins_num
        for p in params:
            if p.dtype != torch.float32 or not p.is_cuda or not p.is_contiguous() or p.device.index != self.index:
                raise RuntimeError("DM_NeRF parameters must be contiguous float32 tensors on cuda:%d" % self.index)
        self._bound[slot] = None       # a pack that fails leaves the slot unbound
        self.call("dmnerf_set_weights", self.handle, slot, _lib.ptrs(params), len(params), ins_num)
        self._bound[slot] = key
        self._keepalive[slot] = params
        return ins_num

    def call(self, name, *args):
        """Call the status-returning entry point `name` with `args` and the current stream; RuntimeError on a non-zero
        status, with the library's message."""
        _lib.check(getattr(self.lib, name)(*args, self.stream()), name)

    def sync_check(self):
        """Synchronise the current stream and raise if any native kernel reported an asynchronous failure."""
        self.call("dmnerf_sync_check", self.handle)

    def slot_for(self, model):
        """Slot to evaluate `model` alone (DM_NeRF.forward): reuse a slot it already occupies."""
        for s in (1, 0):
            if self._bound[s] is not None and self._bound[s][0] == id(model):
                return s
        return 0

    def close(self):
        if self.handle:
            self.lib.dmnerf_ctx_destroy(self.handle)
            self.handle = None
