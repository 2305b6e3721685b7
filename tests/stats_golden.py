"""Replays tests/golden/stats_*.npz (reference metrics outcomes, oracle/gen_golden_stats.py) against the mirror in
hover_net_b200.metrics / hover_net_b200.compute_stats, with whatever pair-table source is installed."""
import builtins
import json
import os
import warnings

import numpy as np
import pytest
import scipy.io as sio

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def load(name):
    return np.load(os.path.join(GOLD, name))


def _same(a, b):
    """== with NaN equal to NaN, recursively over lists; exact (bit-for-bit) for floats."""
    if isinstance(a, list) or isinstance(b, list):
        return isinstance(a, list) and isinstance(b, list) and len(a) == len(b) and all(map(_same, a, b))
    if isinstance(a, float) and isinstance(b, float) and np.isnan(a) and np.isnan(b):
        return True
    return type(a) is type(b) and a == b


def _enc(v):
    if isinstance(v, (list, tuple)):
        return [_enc(x) for x in v]
    if isinstance(v, np.ndarray):
        return [_enc(x) for x in v.tolist()]
    if isinstance(v, (np.integer, int)):
        return int(v)
    return float(v)


def check_stats_utils(S):
    """Every recorded stats_utils call: same value (bit-exact) or same exception class."""
    g = load("stats_utils.npz")
    results = json.loads(str(g["results"]))
    assert len(results) > 150
    for r in results:
        true, pred = g["true_%d" % r["case"]], g["pred_%d" % r["case"]]
        if r["remapped"]:
            true, pred = S.remap_label(true), S.remap_label(pred)
        fn = getattr(S, r["func"])
        what = "%s %s%s" % (r["name"], r["func"], r["args"])
        expect = r.get("mirror") or r.get("raises")
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            if expect:
                with pytest.raises(getattr(builtins, expect)):
                    fn(true, pred, *r["args"])
                continue
            got = _enc(fn(true, pred, *r["args"]))
        assert _same(got, r["value"]), "%s: %r != %r" % (what, got, r["value"])
    for k in ("remap_plain", "remap_by_size"):
        got = S.remap_label(g["remap_in"], by_size=k == "remap_by_size")
        assert got.dtype == np.int32 and np.array_equal(got, g[k]), k
    n = max(r["case"] for r in results)
    assert np.array_equal(S.remap_label(g["pred_%d" % n], by_size=True), g["remap_e2e_by_size"])
    empty = np.zeros((5, 7), np.int64)
    assert S.remap_label(empty) is empty
    for r in (12, 3):
        pairing, ua, ub = S.pair_coordinates(g["pc_a"], g["pc_b"], r)
        for got, key in ((pairing, "pc_pairing_%d"), (ua, "pc_unpaired_a_%d"), (ub, "pc_unpaired_b_%d")):
            ref = g[key % r]
            assert got.dtype == ref.dtype and got.shape == ref.shape and np.array_equal(got, ref), key % r


def check_compute_stats(C, tmp_path, capsys):
    """run_nuclei_inst_stat / run_nuclei_type_stat on the recorded .mat directories: return value and stdout."""
    g = load("stats_compute.npz")
    td, pd = str(tmp_path / "true") + "/", str(tmp_path / "pred") + "/"
    os.makedirs(td)
    os.makedirs(pd)
    for i in range(3):
        sio.savemat(td + "img_%d.mat" % i, {"inst_map": g["true_map_%d" % i], "inst_centroid": g["true_cen_%d" % i],
                                            "inst_type": g["true_type_%d" % i]})
        sio.savemat(pd + "img_%d.mat" % i, {"inst_map": g["pred_map_%d" % i], "inst_centroid": g["pred_cen_%d" % i],
                                            "inst_type": g["pred_type_%d" % i]})
    capsys.readouterr()
    metrics = C.run_nuclei_inst_stat(pd, td)
    out = capsys.readouterr().out
    assert metrics.dtype == g["inst_metrics"].dtype and np.array_equal(metrics, g["inst_metrics"])
    first, rest = out.split("\n", 1)
    assert first == pd and rest == str(g["inst_stdout"])
    assert C.run_nuclei_type_stat(pd, td) is None
    assert capsys.readouterr().out == str(g["type_stdout"])
