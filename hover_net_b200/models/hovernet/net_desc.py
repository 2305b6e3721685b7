"""Drop-in for reference `models/hovernet/net_desc.py`: `create_model` (net_desc.py:149) returns an
object the reference's loader can treat like the torch module it replaces --
`load_state_dict(strict=True)`, `.to()`, `.eval()` -- while the network itself lives in libhvn
(hand-written sm_90a kernels).  `torch.nn.DataParallel(net)` is unnecessary: one process per GPU."""
import numpy as np

from ... import _lib
from ...arch import state_dict_spec


def convert_pytorch_checkpoint(net_state_dict):
    """reference run_utils/utils.py:15-29: a checkpoint saved from `DataParallel` has every key prefixed with
    `module.`; the prefix is stripped only when ALL keys carry it."""
    names = list(net_state_dict.keys())
    if names and all(v.split(".")[0] == "module" for v in names):
        net_state_dict = {".".join(k.split(".")[1:]): v for k, v in net_state_dict.items()}
    return net_state_dict


class HoVerNet(object):
    """precision: "highest" (default) or "high" -- see `_lib.Context`.  An extension: the reference has no such
    argument (its PyTorch convolutions run in TF32 on this GPU by default).
    tta: False (default) or True -- test-time augmentation over the eight dihedral views, see `_lib.Context`.  An
    extension too: the reference has no test-time augmentation."""

    def __init__(self, input_ch=3, nr_types=None, freeze=False, mode="original", device=None, precision="highest",
                 tta=False):
        assert mode == "original" or mode == "fast", \
            "Unknown mode `%s` for HoVerNet %s. Only support `original` or `fast`." % (mode, "")
        assert input_ch == 3, "only RGB input is supported"
        _lib.precision_code(precision)  # ValueError before a context exists
        _lib.tta_code(tta)
        self.mode = mode
        self.freeze = freeze
        self.nr_types = nr_types
        self.output_ch = 3 if nr_types is None else 4
        self.training = False
        if device is None:
            import os
            device = int(os.environ.get("LOCAL_RANK", "0"))
        self.precision = precision
        self.tta = tta
        self.ctx = _lib.Context(device, mode, nr_types, precision=precision, tta=tta)
        self._loaded = False

    # ---- torch.nn.Module look-alikes used by reference infer/base.py:64-70
    def load_state_dict(self, state_dict, strict=True):
        spec = state_dict_spec(self.mode, self.nr_types)
        sd = convert_pytorch_checkpoint(dict(state_dict))
        missing = [k for k in spec if k not in sd and not k.endswith("num_batches_tracked")
                   and k != "upsample2x.unpool_mat"]
        unexpected = [k for k in sd if k not in spec]
        if strict and (missing or unexpected):
            raise RuntimeError("Error(s) in loading state_dict for HoVerNet:\n\tMissing key(s): %s\n\t"
                               "Unexpected key(s): %s" % (missing, unexpected))
        for k, v in sd.items():
            if k not in spec or k.endswith("num_batches_tracked") or k == "upsample2x.unpool_mat":
                continue
            a = v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)
            self.ctx.load_param(k, a)
        self.ctx.finalize_weights()
        self._loaded = True
        return self

    def to(self, *a, **k):
        return self

    def eval(self):
        self.training = False
        return self

    def cuda(self, *a, **k):
        return self

    @property
    def module(self):  # so that code written for DataParallel(net).module keeps working
        return self

    def __call__(self, *a, **k):
        raise RuntimeError("call models.hovernet.run_desc.infer_step(batch, model) -- the fused device path")


def create_model(mode=None, *, precision="highest", tta=False, **kwargs):
    if mode not in ["original", "fast"]:
        assert "Unknown Model Mode %s" % mode
    return HoVerNet(mode=mode, precision=precision, tta=tta, **kwargs)
