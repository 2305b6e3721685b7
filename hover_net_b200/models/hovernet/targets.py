"""Drop-in for reference `models/hovernet/targets.py` (`gen_instance_hv_map`, `gen_targets`), computed on the
device by `hvn_targets` (csrc/targets.cu): bit-identical HV maps, and ValueError for exactly the maps the
reference raises on.  The visualisation helper `prep_sample` is not provided (it needs matplotlib)."""
import numpy as np

from ... import _lib
from .post_proc import _ctx

_FLAG_MESSAGES = (
    (_lib.TG_NO_BACKGROUND, "the instance map has no background (0) pixel"),
    (_lib.TG_NO_BACKGROUND_CROP, "no background (0) pixel is left in the crop once instances of < 30 pixels there "
                                 "are removed"),
    (_lib.TG_EMPTY_BOX, "an instance's box, wrapped at the map edge, holds none of its pixels (its centre of mass "
                        "is NaN)"),
)


def raise_for_flags(flags, names=None):
    """ValueError for the first flagged map (named names[i], or "map i"), for the condition the reference meets
    first."""
    for i, f in enumerate(np.asarray(flags).reshape(-1)):
        for bit, msg in _FLAG_MESSAGES:
            if int(f) & bit:
                raise ValueError("%s: %s" % (names[i] if names else "map %d" % i, msg))


def cropping_center(x, crop_shape, batch=False):
    """Centre crop at offset int((H - crop) * 0.5), as the reference's misc/utils.cropping_center."""
    o = 1 if batch else 0
    h0 = int((x.shape[o] - crop_shape[0]) * 0.5)
    w0 = int((x.shape[o + 1] - crop_shape[1]) * 0.5)
    if batch:
        return x[:, h0:h0 + crop_shape[0], w0:w0 + crop_shape[1]]
    return x[h0:h0 + crop_shape[0], w0:w0 + crop_shape[1]]


def gen_instance_hv_map(ann, crop_shape):
    """Full-size float32 [H,W,2] (x, y) HV map of instance map `ann`; only instances with >= 30 pixels inside the
    centre crop get offsets."""
    hv, flags = _ctx().targets(ann, crop_shape)
    raise_for_flags(flags)
    return hv[0]


def gen_targets(ann, crop_shape, **kwargs):
    """{"hv_map": float32 [h,w,2], "np_map": int32 [h,w] (ann > 0)}, both centre-cropped to crop_shape."""
    hv_map = gen_instance_hv_map(ann, crop_shape)
    np_map = (np.asarray(ann) > 0).astype(np.int32)
    return {
        "hv_map": cropping_center(hv_map, crop_shape),
        "np_map": cropping_center(np_map, crop_shape),
    }
