"""DM_NeRF network with the reference's constructor, parameter names and shapes
(networks/dm_nerf.py:58-106) so checkpoints, `Adam(model.parameters())`, `.to(device)`, `.train()/.eval()`
and `print(model)` behave identically; forward() runs the fused CUDA kernel."""
import torch
import torch.nn as nn

from . import _lib
from .engine import get_context   # noqa: F401
from .synth import layer_table


class DM_NeRF(nn.Module):
    """Parameter container + forward.  The layers are created from synth.layer_table(), whose entries carry the reference's
    state_dict names (`mlps.3`, `rgb_feature_linears.0`, ...): a dotted name becomes a slot of an nn.ModuleList."""

    def __init__(self, D=8, W=256, input_ch_pts=3, input_ch_views=3, skips=[4], ins_num=None):
        super().__init__()
        self.skips, self.input_ch_pts, self.input_ch_views = skips, input_ch_pts, input_ch_views
        if not (D == 8 and W == 256 and input_ch_pts == 63 and input_ch_views == 27 and list(skips) == [4]):
            raise NotImplementedError(
                "the native kernels are specialised for DM_NeRF(D=8, W=256, input_ch_pts=63, input_ch_views=27, "
                "skips=[4]) -- the only configuration config.create_nerf builds (config.py:126-138)")
        if ins_num is None or not (1 <= int(ins_num) <= _lib.N_PARAMS * 0 + 127):
            raise ValueError("ins_num must be in [1, 127], got %r" % (ins_num,))
        # layers are created and registered in table order == the reference's construction order, so the state_dict /
        # optimizer parameter order and the default-init RNG stream are the reference's
        for name, fan_out, fan_in in layer_table(int(ins_num), W, D, input_ch_pts, input_ch_views, tuple(skips)):
            layer = nn.Linear(fan_in, fan_out)
            if "." in name:
                list_name = name.split(".")[0]
                if not hasattr(self, list_name):
                    setattr(self, list_name, nn.ModuleList())
                getattr(self, list_name).append(layer)
            else:
                setattr(self, name, layer)

    @property
    def ins_num(self):
        return self.ins_linear.out_features - 1

    def forward(self, x, impl=_lib.IMPL_AUTO):
        from .autograd import mlp_forward
        return mlp_forward(self, x, impl)
