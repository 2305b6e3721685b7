"""Generates tests/golden/stats_*.npz by running the UNMODIFIED reference metrics (metrics/stats_utils.py,
compute_stats.py) from /root/reference on the CPU.  `matplotlib` (an unused import there) is stubbed.

Run in the build container only (the GPU box has no /root/reference):  python -m oracle.gen_golden_stats

Every input is rebuilt from seeds (hover_net_b200.synth), so the files regenerate with equal arrays.
* stats_utils.npz   : maps true_<k> / pred_<k> and, as JSON in `results`, the reference outcome of every
                      stats_utils function on them (value, pairing lists, or the exception class).  Cases whose ids
                      are not exactly {0..N} carry `mirror: IndexError` for the get_fast_* functions (DESIGN §2).
                      Includes remap_label (area ties) and pair_coordinates outputs.
* stats_compute.npz : two small .mat directories (maps, centroids, types) and the return value and printed
                      lines of run_nuclei_inst_stat / run_nuclei_type_stat on them.
"""
import contextlib
import io
import json
import os
import sys
import tempfile
import types
import warnings

import numpy as np
import scipy.io as sio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden")

from hover_net_b200 import synth  # noqa: E402
from oracle import postproc_oracle as P  # noqa: E402

FAST = ("get_fast_aji", "get_fast_aji_plus", "get_fast_pq", "get_fast_dice_2")


def _import_ref():
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    sys.modules.setdefault("matplotlib", mpl)
    sys.modules.setdefault("matplotlib.pyplot", mpl.pyplot)
    sys.path.insert(0, REF)
    import compute_stats
    from metrics import stats_utils
    return stats_utils, compute_stats


def _enc(v):
    if isinstance(v, (list, tuple)):
        return [_enc(x) for x in v]
    if isinstance(v, np.ndarray):
        return [_enc(x) for x in v.tolist()]
    if isinstance(v, (np.integer, int)):
        return int(v)
    return float(v)


def _run(fn, *args):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            return {"value": _enc(fn(*args))}
        except Exception as e:  # the reference's exception is part of its behaviour
            return {"raises": type(e).__name__}


def _contiguous(m):
    u = np.unique(m)
    return u[0] == 0 and u[-1] == u.size - 1


# ------------------------------------------------------------------------------------------------ inputs
def _perturb(true, kind, seed):
    rng = np.random.default_rng(4000 + seed)
    pred = true.copy()
    n = int(true.max())
    if kind in ("shift", "mixed"):
        pred = np.roll(pred, (2, -3), (0, 1))
    if kind in ("merge", "mixed"):
        for i in range(1, n, 5):  # id i+1 joins id i
            pred[pred == i + 1] = i
    if kind in ("split", "mixed"):
        nxt = n + 1
        for i in range(1, n + 1, 3):
            ys, xs = np.nonzero(pred == i)
            if xs.size:
                cut = (pred == i) & (np.arange(pred.shape[1])[None, :] > int(xs.mean()))
                pred[cut] = nxt
                nxt += 1
    if kind in ("drop", "mixed"):
        for i in rng.choice(np.arange(1, n + 1), max(1, n // 4), replace=False):
            pred[pred == i] = 0
    if kind in ("fp", "mixed"):
        extra = synth.synth_instances(*true.shape, seed=seed + 50, density=1.0 / 600.0)
        add = (extra > 0) & (pred == 0)
        pred[add] = extra[add] + 1000
    return pred.astype(np.int32)


def _tie_maps():
    t = np.zeros((32, 32), np.int32)
    p = np.zeros((32, 32), np.int32)
    t[2:6, 2:10] = 1           # AJI argmax tie: two predictions of IoU 1/2 each
    p[2:6, 2:6] = 1
    p[2:6, 6:10] = 2
    t[10:14, 2:6] = 2          # Munkres tie: 2 x 2 block of equal IoUs (1/3)
    t[10:14, 6:10] = 3
    p[10:12, 2:10] = 3
    p[12:14, 2:10] = 4
    t[20:24, 20:24] = 4        # exact match
    p[20:24, 20:24] = 5
    return t, p


def _cases():
    out = []
    for seed, kind in enumerate(("identity", "shift", "merge", "split", "drop", "fp", "mixed", "mixed")):
        true = synth.synth_instances(96, 96, seed=seed, density=1.0 / 250.0)
        out.append(("%s_%d" % (kind, seed), true, _perturb(true, kind, seed)))
    out.append(("ties",) + _tie_maps())
    z = np.zeros((24, 24), np.int32)
    blob = z.copy()
    blob[3:9, 4:12] = 1
    blob[14:20, 10:16] = 2
    out.append(("both_empty", z, z))
    out.append(("pred_empty", blob, z))
    out.append(("true_empty", z, blob))
    nc = np.zeros((24, 24), np.int32)  # pred ids {1, 3, 4}, id 3 overlapping a true instance
    nc[3:9, 4:8] = 3
    nc[14:20, 10:16] = 1
    nc[0:2, 20:24] = 4
    out.append(("noncontig_pred", blob, nc))
    out.append(("noncontig_true", nc, blob))
    full = np.full((24, 24), 1, np.int32)
    full[12:, :] = 2
    out.append(("no_background_2ids", full, blob))
    out.append(("no_background_1id", np.ones((24, 24), np.int32), blob))
    # end to end: ground truth vs the C oracle's `process` (bit-exact with the device) on the matching pred map
    pm = synth.synth_pred_map(164, 164, None, 2)
    inst, _ = P.process_table(pm, None)
    out.append(("e2e", synth.synth_instances(164, 164, seed=2), inst.astype(np.int32)))
    return out


def gen_stats_utils(S):
    arrays, results = {}, []
    for k, (name, true, pred) in enumerate(_cases()):
        arrays["true_%d" % k] = true
        arrays["pred_%d" % k] = pred
        contiguous = _contiguous(true) and _contiguous(pred)
        if name.startswith(("noncontig", "no_background")) or name in ("both_empty", "pred_empty", "true_empty", "ties"):
            t, p, remapped = true, pred, False  # as given
        else:
            t, p, remapped = S.remap_label(true), S.remap_label(pred), True
            contiguous = True
        calls = [("get_fast_aji", ()), ("get_fast_aji_plus", ()), ("get_fast_dice_2", ()), ("get_dice_1", ()),
                 ("get_dice_2", ())] + [("get_fast_pq", (m,)) for m in (0.3, 0.5, 0.7, 0.0, -0.1)]
        for fn, extra in calls:
            r = {"case": k, "name": name, "remapped": remapped, "func": fn, "args": list(extra)}
            r.update(_run(getattr(S, fn), t, p, *extra))
            if fn in FAST and not contiguous and not (fn == "get_fast_pq" and extra[0] < 0):
                r["mirror"] = "IndexError"
            results.append(r)
        for fn in ("get_dice_1", "get_dice_2"):  # raw ids: these two take any ids
            if remapped:
                r = {"case": k, "name": name, "remapped": False, "func": fn, "args": []}
                r.update(_run(getattr(S, fn), true, pred))
                results.append(r)
    # remap_label with area ties (ids 5 and 9 of equal area, 2 larger, 7 smaller)
    m = np.zeros((20, 20), np.int32)
    m[0:4, 0:4] = 5
    m[6:10, 0:4] = 9
    m[12:18, 0:6] = 2
    m[0:2, 10:13] = 7
    m[15:19, 12:16] = 3
    arrays["remap_in"] = m
    arrays["remap_plain"] = S.remap_label(m, by_size=False)
    arrays["remap_by_size"] = S.remap_label(m, by_size=True)
    k = len(_cases()) - 1
    arrays["remap_e2e_by_size"] = S.remap_label(arrays["pred_%d" % k], by_size=True)
    # pair_coordinates
    rng = np.random.default_rng(77)
    a = rng.uniform(0, 100, (40, 2)).astype(np.float32)
    b = np.concatenate([a[rng.permutation(40)[:30]] + rng.normal(0, 4, (30, 2)), rng.uniform(0, 100, (12, 2))])
    b = b.astype(np.float32)
    arrays["pc_a"], arrays["pc_b"] = a, b
    for r in (12, 3):
        pairing, ua, ub = S.pair_coordinates(a, b, r)
        arrays["pc_pairing_%d" % r], arrays["pc_unpaired_a_%d" % r], arrays["pc_unpaired_b_%d" % r] = pairing, ua, ub
    arrays["results"] = np.array(json.dumps(results))
    np.savez_compressed(os.path.join(OUT, "stats_utils.npz"), **arrays)
    print("stats_utils.npz: %d cases, %d results" % (k + 1, len(results)))


def _mat(m, rng, ntypes=4):
    ids = [i for i in np.unique(m) if i != 0]
    cen = np.array([[np.nonzero(m == i)[1].mean(), np.nonzero(m == i)[0].mean()] for i in ids]).reshape(-1, 2)
    typ = rng.integers(1, ntypes + 1, (len(ids), 1))
    return cen, typ


def gen_compute(C):
    rng = np.random.default_rng(91)
    arrays = {}
    with tempfile.TemporaryDirectory() as d:
        td, pd = os.path.join(d, "true") + "/", os.path.join(d, "pred") + "/"
        os.makedirs(td)
        os.makedirs(pd)
        for i in range(3):
            true = synth.synth_instances(64, 80, seed=20 + i, density=1.0 / 200.0)
            pred = _perturb(true, "mixed", 20 + i)
            tc, tt = _mat(true, rng)
            pc, pt = _mat(pred, rng)
            for key, v in (("true_map", true), ("pred_map", pred), ("true_cen", tc), ("true_type", tt),
                           ("pred_cen", pc), ("pred_type", pt)):
                arrays["%s_%d" % (key, i)] = v
            sio.savemat(td + "img_%d.mat" % i, {"inst_map": true, "inst_centroid": tc, "inst_type": tt})
            sio.savemat(pd + "img_%d.mat" % i, {"inst_map": pred, "inst_centroid": pc, "inst_type": pt})
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            metrics = C.run_nuclei_inst_stat(pd, td, print_img_stats=False)
        arrays["inst_metrics"] = np.asarray(metrics)
        arrays["inst_stdout"] = np.array(buf.getvalue().split("\n", 1)[1])  # first line is pred_dir
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            C.run_nuclei_type_stat(pd, td)
        arrays["type_stdout"] = np.array(buf.getvalue())
    np.savez_compressed(os.path.join(OUT, "stats_compute.npz"), **arrays)
    print("stats_compute.npz:", arrays["inst_stdout"], arrays["type_stdout"])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    P.build()
    S, C = _import_ref()
    gen_stats_utils(S)
    gen_compute(C)
