"""Per-nucleus measurements without a GPU: the float64 restatement (tests/features_ref.py) against cv2's own
contourArea, arcLength, convexHull and moments; the column names against include/hvn.h; the --save_features flags; and
the tile-mode writers with and without features."""
import json
import os
import re

import numpy as np
import pytest

import features_ref as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _maps():
    return F.edge_maps() + [("seeded%d" % s, F.seeded_map(96, 128, s)) for s in range(3)]


@pytest.mark.parametrize("name,inst", _maps(), ids=[n for n, _ in _maps()])
def test_restatement_equals_cv2(name, inst):
    import cv2
    table = F.table_of(inst)
    pts, offs = F.cv2_contours(inst, table)
    for k, r in enumerate(table):
        iid, rmin, cmin, rmax, cmax = (int(v) for v in r[:5])
        P = pts[offs[k]:offs[k + 1]]
        c = P.reshape(-1, 1, 2)
        assert F.arc_length(P) == cv2.arcLength(c, True)
        assert abs(F.shoelace2(P)) * 0.5 == cv2.contourArea(c)
        hull = np.array(F.hull(P), dtype=np.int32).reshape(-1, 1, 2)
        cvh = cv2.convexHull(c)
        assert (abs(F.shoelace2(hull.reshape(-1, 2))) * 0.5 if len(hull) >= 3 else 0.0) == cv2.contourArea(cvh)
        # every cv2 hull vertex is one of ours (cv2 may keep collinear points; ours are the strict vertices)
        assert set(map(tuple, hull.reshape(-1, 2).tolist())) <= set(map(tuple, cvh.reshape(-1, 2).tolist()))
        crop = inst[rmin:rmax, cmin:cmax] == iid
        A, m10, m01, mu20, mu11, mu02 = F.moments(crop)
        mo = cv2.moments(crop.astype(np.uint8), binaryImage=True)
        assert (A, m10, m01) == (mo["m00"], mo["m10"], mo["m01"])
        assert (mu20, mu11, mu02) == (mo["mu20"], mo["mu11"], mo["mu02"])  # bit for bit
        d2 = ((P[:, None, :].astype(np.int64) - P[None, :, :]) ** 2).sum(-1)
        assert F.row_features(inst, r, P)[10] == np.sqrt(float(d2.max()))  # feret_max: max over all point pairs


def test_std_numerator_is_exact():
    """Population std of u8 extremes: all 0 and all 255 give exactly 0, a 0/255 half split exactly 127.5."""
    inst = np.zeros((4, 6), np.int32)
    inst[:, :] = 1
    table = F.table_of(inst)
    pts, offs = F.cv2_contours(inst, table)
    for v, want in ((0, 0.0), (255, 0.0)):
        img = np.full((4, 6, 3), v, np.uint8)
        f = F.features(inst, table, pts, offs, img=img)[0]
        assert f[14] == f[15] == f[16] == want and f[11] == float(v)
    img = np.zeros((4, 6, 3), np.uint8)
    img[:, :3] = 255
    assert F.features(inst, table, pts, offs, img=img)[0][14] == 127.5


def test_names_match_header():
    from hover_net_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "hvn.h")).read()
    body = re.search(r"enum\s*\{\s*(HVN_FEAT_AREA[^}]*)\}", hdr).group(1)
    names = [re.sub(r"\s*=.*", "", t.strip())[len("HVN_FEAT_"):].lower() for t in body.split(",") if t.strip()]
    assert tuple(names) == _lib.FEATURE_NAMES == F.NAMES
    assert int(re.search(r"#define HVN_FEAT_LEN (\d+)", hdr).group(1)) == len(names) == _lib.FEAT_LEN


def test_cli_save_features_flags():
    from hover_net_b200 import run_infer
    base = ["--model_path=m.tar"]
    for sub in (["tile", "--input_dir=i", "--output_dir=o"], ["wsi", "--input_dir=i", "--output_dir=o"]):
        _, _, rargs, _ = run_infer.parse(base + sub)
        assert "save_features" not in rargs  # the reference's run_args, unchanged
        _, _, rargs, _ = run_infer.parse(base + sub + ["--save_features"])
        assert rargs["save_features"] is True


def _writer(tmp_path, save_features):
    from hover_net_b200.infer import tile

    class M:
        output_dir = str(tmp_path)
        nr_types = None
        save_raw_map = save_qupath = draw_dot = False
        type_info_dict = {None: ["no label", [0, 0, 0]]}
        _save_json = tile.InferManager._save_json
        _write_files = tile.InferManager._write_files

    m = M()
    m.save_features = save_features
    for sub in ("json", "mat", "overlay"):
        os.makedirs(os.path.join(str(tmp_path), sub), exist_ok=True)
    return m


def _info(features):
    from hover_net_b200.models.hovernet.post_proc import table_to_dict
    inst = F.seeded_map(40, 50, 7, n=6)
    table = F.table_of(inst)
    pts, offs = F.cv2_contours(inst, table)
    feats = None
    if features:
        img = np.random.default_rng(1).integers(0, 256, inst.shape + (3,), dtype=np.uint8)
        feats = F.features(inst, table, pts, offs, img=img)
        feats[:, 17] = 0.25  # a stand-in NP mean
    return inst, table_to_dict(table, offs, pts, None, feats), feats


def test_writers_without_features_unchanged(tmp_path):
    """Without save_features the JSON is byte for byte what the writer wrote before features existed, and the .mat
    holds the same variables with the same bytes after the header (which carries a timestamp)."""
    import scipy.io as sio
    inst, info, _ = _info(False)
    img = np.zeros(inst.shape + (3,), np.uint8)
    m = _writer(tmp_path, False)
    m._write_files([("x/a.png", img)], [(None, inst, info)])
    nuc = {int(k): {kk: (vv.tolist() if isinstance(vv, np.ndarray) else vv) for kk, vv in v.items()}
           for k, v in info.items()}
    assert open(str(tmp_path / "json" / "a.json")).read() == json.dumps({"mag": None, "nuc": nuc})
    vals = list(info.values())
    ref = str(tmp_path / "ref.mat")
    sio.savemat(ref, {"inst_map": inst, "inst_uid": np.array(list(info.keys()))[:, None],
                      "inst_centroid": np.array([v["centroid"] for v in vals])})
    assert open(ref, "rb").read()[128:] == open(str(tmp_path / "mat" / "a.mat"), "rb").read()[128:]


def test_writers_with_features(tmp_path):
    import scipy.io as sio
    from hover_net_b200 import _lib
    inst, info, feats = _info(True)
    img = np.zeros(inst.shape + (3,), np.uint8)
    m = _writer(tmp_path, True)
    m._write_files([("x/a.png", img)], [(None, inst, info)])
    js = json.load(open(str(tmp_path / "json" / "a.json")))["nuc"]
    mat = sio.loadmat(str(tmp_path / "mat" / "a.mat"))
    uid = mat["inst_uid"].ravel()
    assert mat["inst_features"].shape == (len(info), _lib.FEAT_LEN)
    assert [str(np.ravel(s)[0]).strip() for s in mat["inst_feature_names"].ravel()] == list(_lib.FEATURE_NAMES)
    table = F.table_of(inst)
    for k, iid in enumerate(uid):
        row = feats[list(table[:, 0]).index(iid)]
        assert np.array_equal(mat["inst_features"][k], row)
        assert js[str(iid)]["features"] == dict(zip(_lib.FEATURE_NAMES, row.tolist()))


def test_features_dict_drops_uncomputed_columns():
    from hover_net_b200.models.hovernet.post_proc import features_dict
    row = np.arange(18, dtype=np.float64)
    row[11:17] = np.nan
    d = features_dict(row)
    assert "mean_r" not in d and "std_b" not in d and d["np_prob_mean"] == 17.0 and len(d) == 12
