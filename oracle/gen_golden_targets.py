"""Generates tests/golden/targets_cases.npz and tests/golden/valid_scalars.npz by running the UNMODIFIED reference
`gen_targets` / `gen_instance_hv_map` (models/hovernet/targets.py, with dataloader/augs.py fix_mirror_padding) and
`proc_valid_step_output` (models/hovernet/run_desc.py) from /root/reference on the CPU.

Run in the build container only (the GPU box has no /root/reference):  python -m oracle.gen_golden_targets

Stubs, none of which changes what is measured:
* `matplotlib` (imported by the reference modules, used only for visualisation) is an empty module, and
  run_desc.viz_step_output is replaced by a function returning None (its figure is not part of the scalars);
* scikit-image is absent, so `skimage.morphology.remove_small_objects` is the reference's own copy in
  misc/utils.py, applied to a copy of the array (skimage returns a new array).  Like the watershed, the goldens are
  therefore not pinned against skimage itself.
* `cv2`, `imgaug` and `torch.utils.data` are not needed by the functions run here.

Every input is rebuilt from seeds (hover_net_b200.synth and numpy generators), so the files regenerate equal.
* targets_cases.npz: ann_<k> int32 [H,W], crop_<k> int32 [2], and either hv_<k> float32 [H,W,2] (full-size
  gen_instance_hv_map output), tgt_hv_<k> / tgt_np_<k> (gen_targets output) or, in `results` (JSON), the class
  of the exception the reference raised.
* valid_scalars.npz: in `results`, for the seeded raw dicts `_raw(*VALID_CASES[k], k)`, nr_types and every
  `track_dict["scalar"]` value (as float64, with the numpy type name) of proc_valid_step_output.
"""
import json
import os
import sys
import types
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden")

from hover_net_b200 import synth  # noqa: E402


def _import_ref():
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    mpl.cm = types.ModuleType("matplotlib.cm")
    for name, mod in (("matplotlib", mpl), ("matplotlib.pyplot", mpl.pyplot), ("matplotlib.cm", mpl.cm)):
        sys.modules.setdefault(name, mod)
    sys.path.insert(0, REF)
    import misc.utils as mu
    sk = types.ModuleType("skimage")
    morph = types.ModuleType("skimage.morphology")
    morph.remove_small_objects = lambda ar, min_size=64, connectivity=1: mu.remove_small_objects(
        ar.copy(), min_size, connectivity)
    sk.morphology = morph
    sys.modules.setdefault("skimage", sk)
    sys.modules.setdefault("skimage.morphology", morph)
    from models.hovernet import targets
    from models.hovernet import run_desc
    run_desc.viz_step_output = lambda raw, nr_types=None: None
    return targets, run_desc


# ------------------------------------------------------------------------------------------------ target maps
def _split_ids(inst, k):
    """Ids merged k to one: the same id in several disjoint pieces."""
    return np.where(inst > 0, (inst + k - 1) // k, 0).astype(np.int32)


def _edge_maps():
    """64 x 64 maps, crop 40 x 40 (rows / cols 12..51): every edge and wrap case of the sliced box."""
    cases = []
    z = lambda: np.zeros((64, 64), np.int32)  # noqa: E731
    a = z()
    a[0:31, 20:27] = 1     # starts in row 0, ends far from the bottom: box rows [62, 33) is empty -> skipped
    a[1:31, 30:37] = 2     # starts in row 1: box rows [63, 33) -> skipped
    a[0:64, 40:44] = 3     # row 0 .. row 63: box rows [62, 64) -> offsets from the last two rows only
    a[20:40, 0:30] = 4     # same in the columns: starts in column 0 and ends far away -> skipped
    a[45:50, 14:20] = 5    # ordinary instance
    cases.append(("wrap_rows", a, (40, 40)))
    b = z()
    b[0:63, 20:26] = 1     # ends in row 62 (exclusive 63): box rows [62, 64) holds row 62 only
    b[30:36, 0:64] = 2     # full width: box cols [62, 64)
    b[50:55, 30:40] = 3
    cases.append(("wrap_edges", b, (40, 40)))
    c = z()
    c[:, 63] = 1           # L plus a bar through the crop: rmin = cmin = 0, box [62, 64) x [62, 64)
    c[63, :] = 1
    c[30, 10:64] = 1
    c[40:45, 20:30] = 2
    cases.append(("wrap_both", c, (40, 40)))
    d = z()
    d[0:62, 20:26] = 1     # ends in row 61: the wrapped box [62, 64) holds none of its pixels -> NaN
    cases.append(("wrap_nan", d, (40, 40)))
    e = z()
    e[5:17, 20:26] = 1     # rows 12..16 inside the crop: exactly 5 * 6 = 30 px -> kept
    e[5:17, 30:36] = 2
    e[16, 35] = 0          # 29 px inside -> removed (NP only)
    e[40:60, 40:60] = 3    # crosses the crop's bottom-right corner
    e[30:34, 14:18] = 4    # 16 px, all inside -> removed
    cases.append(("crop_size", e, (40, 40)))
    f = z()
    f[10:20, 10:20] = 7    # one id, four pieces; two of them touch diagonally only (separate 4-components)
    f[30:40, 30:40] = 7
    f[40:45, 40:45] = 7
    f[45:50, 45:50] = 7
    f[20:30, 40:50] = 3
    f[22:28, 50:60] = 3    # touches the first piece of id 3: same component
    cases.append(("pieces", f, (40, 40)))
    g = z()
    g[20:40, 25:45] = 9
    cases.append(("one_instance", g, (40, 40)))
    cases.append(("empty", z(), (40, 40)))
    h = np.ones((64, 64), np.int32)
    cases.append(("no_background", h, (40, 40)))
    i = np.ones((64, 64), np.int32)
    i[:, 32:] = 2
    cases.append(("no_background_two", i, (40, 40)))
    j = z()
    j[8:56, 8:56] = 4      # the crop is covered by one instance: no background left in it
    cases.append(("no_background_crop", j, (40, 40)))
    k = z()
    k[8:56, 8:56] = 4
    k[12:14, 12:30] = 0    # ... and with background that survives
    k[30:32, 30:32] = 5    # a 4 px instance inside the crop: removed, so the crop has background again
    cases.append(("crop_small_only", k, (40, 40)))
    m = z()
    m[8:56, 8:56] = 4
    m[30:32, 30:32] = 0    # background hole in the crop
    m[29:33, 34:38] = 0
    cases.append(("crop_hole", m, (40, 40)))
    return cases


def _target_cases():
    cases = []
    for (H, crop, seed) in ((270, 80, 1), (256, 164, 2), (540, 164, 3)):
        cases.append(("synth_%d_%d" % (H, crop), synth.synth_instances(H, H, seed=seed), (crop, crop)))
    for k in (2, 3, 5):
        cases.append(("split_%d" % k, _split_ids(synth.synth_instances(270, 270, seed=10 + k), k), (80, 80)))
    cases.append(("dense_270", synth.synth_instances(270, 270, seed=7, density=1.0 / 300.0), (80, 80)))
    cases.append(("rect_96x80", synth.synth_instances(96, 80, seed=8, density=1.0 / 150.0), (61, 47)))
    return cases + _edge_maps()


def _targets(T):
    arrays, results = {}, []
    for k, (name, ann, crop) in enumerate(_target_cases()):
        ann = np.ascontiguousarray(ann, dtype=np.int32)
        arrays["ann_%d" % k] = ann
        arrays["crop_%d" % k] = np.array(crop, np.int32)
        rec = {"name": name}
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            try:
                hv = T.gen_instance_hv_map(ann.copy(), list(crop))
                tgt = T.gen_targets(ann.copy(), list(crop))
            except Exception as e:  # the reference's exception is part of its behaviour
                rec["raises"] = type(e).__name__
            else:
                assert hv.dtype == np.float32 and hv.shape == ann.shape + (2,)
                arrays["hv_%d" % k] = hv
                arrays["tgt_hv_%d" % k] = tgt["hv_map"]
                arrays["tgt_np_%d" % k] = tgt["np_map"]
        results.append(rec)
    arrays["results"] = np.array(json.dumps(results))
    return arrays


# ------------------------------------------------------------------------------------------------ valid scalars
def _raw(n, hw, nr_types, seed):
    rng = np.random.default_rng(6000 + seed)
    prob = rng.random((n, hw, hw), dtype=np.float32)
    prob[:, :4, :4] = 0.5                                     # exactly at the threshold: not foreground
    prob[:, 4:6, :4] = np.nextafter(np.float32(0.5), np.float32(1))
    true_np = (rng.random((n, hw, hw)) < 0.4).astype(np.int32)
    raw = {
        "imgs": rng.integers(0, 256, (n, 8, 8, 3), dtype=np.uint8),
        "true_np": true_np,
        "true_hv": rng.uniform(-1, 1, (n, hw, hw, 2)).astype(np.float32),
        "prob_np": prob,
        "pred_hv": rng.uniform(-1.2, 1.2, (n, hw, hw, 2)).astype(np.float32),
    }
    if nr_types is not None:
        raw["true_tp"] = rng.integers(0, nr_types, (n, hw, hw)).astype(np.int32)
        raw["pred_tp"] = rng.integers(0, nr_types, (n, hw, hw)).astype(np.float32)
    return raw


VALID_CASES = ((3, 80, None), (4, 80, 5), (2, 164, 6), (1, 80, 5))


def _valid(R):
    arrays, results = {}, []
    np.random.seed(0)  # the reference draws the indices of its (stubbed) figure from the global generator
    for k, (n, hw, nt) in enumerate(VALID_CASES):
        raw = _raw(n, hw, nt, k)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            scal = R.proc_valid_step_output(raw, nr_types=nt)["scalar"]
        results.append({"nr_types": nt,
                        "scalar": {key: [float(v), type(v).__name__] for key, v in scal.items()}})
    arrays["results"] = np.array(json.dumps(results))
    return arrays


def main():
    T, R = _import_ref()
    np.savez_compressed(os.path.join(OUT, "targets_cases.npz"), **_targets(T))
    np.savez_compressed(os.path.join(OUT, "valid_scalars.npz"), **_valid(R))
    print("wrote", OUT)


if __name__ == "__main__":
    main()
