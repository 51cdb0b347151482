"""The torch interpreter of the IR (oracle/plan_interp.py) with the rule it lacks: average pooling with
``count_include_pad=False`` (ir.py sets ``exclude_pad`` on such ``avgpool2d`` nodes), where every window is divided by
its taps inside the image.  aten's own pooling with ``count_include_pad=False`` is the executable specification."""
import torch
import torch.nn.functional as F

from oracle.plan_interp import Interp as _Interp


class Interp(_Interp):
    def _avg(self, n, t):
        at = n.attrs
        if not at.get("exclude_pad"):
            return super()._avg(n, t)
        return F.avg_pool2d(t, at["kernel"], at["stride"], at["padding"], False, False, None)

    def _avg_bw(self, n, g):
        at = n.attrs
        if not at.get("exclude_pad"):
            return super()._avg_bw(n, g)
        ref = torch.zeros(n.ins[0].shape, dtype=self.dtype, device=g.device)
        return torch.ops.aten.avg_pool2d_backward(g.contiguous(), ref, list(at["kernel"]), list(at["stride"]),
                                                  list(at["padding"]), False, False, None)
