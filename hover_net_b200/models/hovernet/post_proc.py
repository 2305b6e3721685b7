"""Drop-in for reference `models/hovernet/post_proc.py:94-186` (`process`).

Module-level and picklable like the reference's (it is shipped to pool workers under `spawn`,
infer/tile.py:353-363); each process lazily opens its own post-processing context on
`HVN_DEVICE` / `LOCAL_RANK` / device 0.  Contours are traced on the device (csrc/contour.cu, SURVEY.md
row f3): point for point the reference's cv2.findContours(..., RETR_TREE, CHAIN_APPROX_SIMPLE)[0][0] on the
bbox crop (:133-143); centroids come from the instance table's exact integer sums, evaluated in the
reference's float order (m10/m00 + cmin, :144-152).

Extension the reference lacks: `process_features` is `process` (with centroids) plus each nucleus's shape and intensity
measurements (`_lib.FEATURE_NAMES`, hvn_inst_features, computed on the device) as `inst_info[id]["features"]`.
`process` itself keeps the reference's signature: it is the plugin seam."""
import os

import numpy as np

from ... import _lib

_CTX = {}


def _ctx():
    dev = int(os.environ.get("HVN_DEVICE", os.environ.get("LOCAL_RANK", "0")))
    key = (os.getpid(), dev)
    if key not in _CTX:
        _CTX[key] = _lib.Context(dev)
    return _CTX[key]


def features_dict(row):
    """One hvn_inst_features row -> {name: value} over _lib.FEATURE_NAMES, without the columns that were not computed
    (NaN: no image or no prediction map was given)."""
    return {k: float(v) for k, v in zip(_lib.FEATURE_NAMES, row) if not np.isnan(v)}


def table_to_dict(table, offs, pts, nr_types, feats=None):
    """Instance table rows + device-traced contours -> the reference's inst_info_dict (post_proc.py:120-181).
    table [n,10], offs [>= n+1] (point range of row r = pts[offs[r]:offs[r+1]]), pts [total,2] (x, y).  With feats
    (hvn_inst_features rows [n,FEAT_LEN]) every entry gains "features" (features_dict)."""
    info = {}
    for k, r in enumerate(table):
        iid, rmin, cmin, rmax, cmax, area, sx, sy, tp, tc = (int(v) for v in r)
        cnt = pts[int(offs[k]) : int(offs[k + 1])]
        if cnt.shape[0] < 3:  # < 3 points dont make a contour (:140-143; a 1-point contour squeezes to 1-D there)
            continue
        # cv2.moments of the bbox crop: m00 = area, m10 = sum(x - cmin), m01 = sum(y - rmin) -- exact integers
        cen = np.array([float(sx - cmin * area) / float(area), float(sy - rmin * area) / float(area)])
        cen[0] += cmin
        cen[1] += rmin
        info[iid] = {"bbox": np.array([[rmin, cmin], [rmax, cmax]]), "centroid": cen, "contour": np.array(cnt, dtype=np.int32),
                     "type_prob": None, "type": None}
        if nr_types is not None:
            info[iid]["type"] = int(tp)
            info[iid]["type_prob"] = float(tc / (area + 1.0e-6))
        if feats is not None:
            info[iid]["features"] = features_dict(feats[k])
    return info


def process(pred_map, nr_types=None, return_centroids=False):
    """pred_map [H,W,C] -> (pred_inst int32 [H,W], inst_info_dict or None)."""
    return _process(pred_map, nr_types, return_centroids, None, False)


def process_features(pred_map, nr_types=None, image=None):
    """`process(pred_map, nr_types, return_centroids=True)` with every entry of the dict gaining "features": the
    measurements of the nucleus on pred_inst, on `image` (RGB u8 [H,W,3]; without it the colour columns are left out)
    and on pred_map's NP channel."""
    return _process(pred_map, nr_types, True, image, True)


def _process(pred_map, nr_types, return_centroids, image, features):
    pm = np.asarray(pred_map)
    if nr_types is not None:
        # reference: pred_type = pred_map[..., :1].astype(int32); pred_inst = pred_map[..., 1:]
        if pm.shape[-1] != 4:
            raise ValueError("typed post-processing expects [tp, np, hv_x, hv_y] channels")
    elif pm.shape[-1] != 3:
        raise ValueError("seg-only post-processing expects [np, hv_x, hv_y] channels")
    if image is not None and np.asarray(image).shape != pm.shape[:2] + (3,):
        raise ValueError("image must be RGB [H,W,3] of the map's size, got %s" % (np.asarray(image).shape,))
    if not (return_centroids or features or nr_types is not None):
        inst, table, nrows = _ctx().postproc(pm.astype(np.float32, copy=False), nr_types)
        return inst[0], None
    pm = pm.astype(np.float32, copy=False)
    inst, table, nrows, offs, pts = _ctx().postproc_contours(pm, nr_types)
    n = int(nrows[0])
    feats = None
    if features:
        feats = _ctx().inst_features(inst[0], table[0, :n], pts, offs[: n + 1], image=image, pred=pm)
    info = table_to_dict(table[0, :n], offs, pts, nr_types, feats)
    return inst[0], info
