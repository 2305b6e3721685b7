"""Numpy restatement of the device HV targets (csrc/targets.cu), written from the semantics of the reference's
`gen_instance_hv_map` after `fix_mirror_padding`, not from its code:

* every 4-connected component of equal non-zero id is one instance (the reference gives every later piece of an
  id a fresh id, so ids and components correspond one to one);
* an instance gets offsets only when >= 30 of its pixels lie inside the centre crop (`cropping_center` offsets
  int((H - crop) * 0.5));
* its full-map extent (exclusive max) is expanded by 2 and taken with Python slice semantics; a side < 2 skips it;
* centre of mass over its pixels inside that box: integer sums, one float64 division, int(com + 0.5);
* offsets 1..len - com, negatives divided by -min and positives by max in float32; only its own pixels are written.

`hv_map(ann, crop_shape)` -> (hv float32 [H,W,2] (x, y), flags) with the HVN_TG_* bits of include/hvn.h: 1 no
background in the map, 2 no background left in the crop, 4 a box without any of its instance's pixels.  Raises
ValueError on a negative id and when max id + number of components exceeds 2^31 - 1 (the device reports both as
HVN_ERR_INVALID)."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

NO_BACKGROUND, NO_BACKGROUND_CROP, EMPTY_BOX = 1, 2, 4
MIN_IN_CROP = 30
INT32_MAX = 2 ** 31 - 1


def components(ann):
    """Component label [H,W] (-1 on background, 0..K-1 elsewhere) and K."""
    H, W = ann.shape
    idx = np.arange(H * W).reshape(H, W)
    fg = ann > 0
    right = fg[:, :-1] & (ann[:, :-1] == ann[:, 1:])
    down = fg[:-1, :] & (ann[:-1, :] == ann[1:, :])
    a = np.concatenate([idx[:, :-1][right], idx[:-1, :][down]])
    b = np.concatenate([idx[:, 1:][right], idx[1:, :][down]])
    g = coo_matrix((np.ones(a.size, np.int8), (a, b)), shape=(H * W, H * W))
    _, lab = connected_components(g, directed=False)
    u, inv = np.unique(lab.reshape(H, W)[fg], return_inverse=True)
    out = np.full((H, W), -1, np.int64)
    out[fg] = inv
    return out, int(u.size)


def hv_map(ann, crop_shape):
    ann = np.asarray(ann)
    if (ann < 0).any():
        raise ValueError("negative instance id")
    H, W = ann.shape
    comp, K = components(ann)
    if int(ann.max(initial=0)) + K > INT32_MAX:
        raise ValueError("largest id + number of components exceeds 2^31 - 1")
    h0, w0 = int((H - crop_shape[0]) * 0.5), int((W - crop_shape[1]) * 0.5)
    crop = comp[h0:h0 + crop_shape[0], w0:w0 + crop_shape[1]]
    in_crop = np.bincount(crop[crop >= 0], minlength=K)
    flags = 0
    if not (ann == 0).any():
        flags |= NO_BACKGROUND
    if not ((crop < 0).any() or (in_crop < MIN_IN_CROP)[crop[crop >= 0]].any()):
        flags |= NO_BACKGROUND_CROP
    hv = np.zeros((H, W, 2), np.float32)
    ys, xs = np.nonzero(comp >= 0)
    c = comp[ys, xs]
    rmin = np.full(K, H, np.int64)
    cmin = np.full(K, W, np.int64)
    rmax = np.zeros(K, np.int64)
    cmax = np.zeros(K, np.int64)
    np.minimum.at(rmin, c, ys)
    np.minimum.at(cmin, c, xs)
    np.maximum.at(rmax, c, ys + 1)
    np.maximum.at(cmax, c, xs + 1)
    for k in np.nonzero(in_crop >= MIN_IN_CROP)[0]:
        r0, r1, _ = slice(int(rmin[k]) - 2, int(rmax[k]) + 2).indices(H)
        c0, c1, _ = slice(int(cmin[k]) - 2, int(cmax[k]) + 2).indices(W)
        if r1 - r0 < 2 or c1 - c0 < 2:
            continue
        by, bx = np.nonzero(comp[r0:r1, c0:c1] == k)
        if by.size == 0:
            flags |= EMPTY_BOX
            continue
        coms = [int(int(v.sum()) / by.size + 0.5) for v in (by, bx)]
        for ch, (v, com) in enumerate(((bx, coms[1]), (by, coms[0]))):
            f = (v + 1 - com).astype(np.float32)
            neg, pos = f < 0, f > 0
            if neg.any():
                f[neg] = f[neg] / np.float32(-f[neg].min())
            if pos.any():
                f[pos] = f[pos] / np.float32(f[pos].max())
            hv[r0 + by, c0 + bx, ch] = f
    return hv, flags
