"""Benchmark of the instance metrics (hvn_inst_pairs + hover_net_b200.metrics / compute_stats) on the H100.

    python tools/bench_stats.py --out DIR [--reps 20]

Workloads: 14 maps of 1000 x 1000 at ~1/900 px^-2 nuclei density (about the CoNSeP test set) and one 4096 x 4096
map, with predictions shifted, relabelled and thinned.  Reports, as JSON in DIR/bench_stats.json:
* the hvn_inst_pairs_dev call time per map (CUDA events on the context stream, around the whole call including
  its 12-byte status read-back), and the bandwidth of 8 B read per pixel over that time against the HBM3 peak;
* the host finishing time of each metric per image, and run_nuclei_inst_stat end to end per image;
* that every timed table equals the numpy oracle's;
* the card name, power limit and max SM clock (nvidia-smi query) read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import scipy.io as sio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hover_net_b200 import compute_stats, synth  # noqa: E402
from hover_net_b200.metrics import stats_utils as S  # noqa: E402
from hover_net_b200.models.hovernet.post_proc import _ctx  # noqa: E402
from oracle import stats_oracle as O  # noqa: E402

HBM_PEAK = 3.35e12  # H100 SXM data sheet


def _peak():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        try:
            v = json.load(open(path)).get("hbm_bytes_per_s")
            if v:
                return float(v), "MEASURED_PEAKS.json"
        except (ValueError, AttributeError):
            pass
    return HBM_PEAK, "H100 SXM data sheet"


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def _pred_of(true, seed):
    rng = np.random.default_rng(seed)
    p = np.roll(true, (2, -3), (0, 1))
    ids = np.arange(int(p.max()) + 1)
    keep = rng.uniform(0, 1, ids.size) > 0.1  # drop ~10 % of the instances
    keep[0] = True
    lut = np.where(keep, ids + 11, 0)
    lut[0] = 0
    return lut[p].astype(np.int32)


def _time_dev(ctx, t, p, reps):
    n, H, W = t.shape
    ref_rows, ref_offs = O.pair_table(t, p)
    cap = int(ref_offs[-1])
    bufs = [ctx.malloc(b) for b in (t.nbytes, p.nbytes, 24 * max(cap, 1), 8 * (n + 1))]
    d_t, d_p, d_rows, d_offs = bufs
    try:
        ctx.h2d(d_t, t, t.nbytes)
        ctx.h2d(d_p, p, p.nbytes)
        for _ in range(3):
            assert ctx.inst_pairs_dev(d_t, d_p, n, H, W, d_rows, cap, d_offs)
        ms = []
        for _ in range(reps):
            ctx.timer_start()
            ctx.inst_pairs_dev(d_t, d_p, n, H, W, d_rows, cap, d_offs)
            ms.append(ctx.timer_stop())
        offs = np.zeros(n + 1, np.int64)
        rows = np.zeros((cap, 3), np.int64)
        ctx.d2h(offs, d_offs, offs.nbytes)
        ctx.d2h(rows, d_rows, rows.nbytes)
        ctx.sync()
    finally:
        for d in bufs:
            ctx.free(d)
    m = np.repeat(np.arange(n), np.diff(offs))
    rows = rows[np.lexsort((rows[:, 1], rows[:, 0], m))]
    equal = bool(np.array_equal(offs, ref_offs) and np.array_equal(rows, ref_rows))
    return np.array(ms), equal, cap


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    ctx = _ctx()
    peak, peak_src = _peak()
    res = {"card": _card(), "hbm_peak_bytes_per_s": peak, "hbm_peak_source": peak_src}

    t0 = time.time()
    conse = np.stack([synth.tiled_instances(1000, 1000, block=250, seed=s, n_unique=8) for s in range(14)])
    big = synth.tiled_instances(4096, 4096, seed=99)[None]
    res["input_build_s"] = time.time() - t0
    for name, t in (("14x1000x1000", conse), ("1x4096x4096", big)):
        p = np.stack([_pred_of(t[i], i) for i in range(t.shape[0])])
        ms, equal, pairs = _time_dev(ctx, t, p, args.reps)
        px = t.size
        res[name] = {"instances_true": int(sum(int(x.max()) for x in t)), "pairs": pairs,
                     "call_ms_median": float(np.median(ms)), "call_ms_min": float(ms.min()),
                     "call_ms_per_map_median": float(np.median(ms)) / t.shape[0],
                     "bytes_read": 8 * px,
                     "bandwidth_bytes_per_s_median": 8 * px / (np.median(ms) * 1e-3),
                     "fraction_of_hbm_peak": 8 * px / (np.median(ms) * 1e-3) / peak,
                     "table_equals_oracle": equal}
        print(name, json.dumps(res[name]))

    # host finishing per metric, one 1000 x 1000 image (table of the raw maps, ids renamed as remap_label would)
    rows, _ = S.pair_table(conse[0], _pred_of(conse[0], 0))
    tab = S._Pairs(rows, conse[0].size).renamed()
    fin = {}
    for name, fn in (("dice_1", lambda: S._dice_1(tab)), ("aji", lambda: S._aji(tab)),
                     ("pq_0.5", lambda: S._pq(tab, 0.5, (np.int32, np.int32))),
                     ("pq_0.3_munkres", lambda: S._pq(tab, 0.3, (np.int32, np.int32))),
                     ("aji_plus", lambda: S._aji_plus(tab)), ("fast_dice_2", lambda: S._fast_dice_2(tab))):
        fn()
        t1 = time.perf_counter()
        for _ in range(5):
            fn()
        fin[name] = (time.perf_counter() - t1) / 5
    res["host_finish_s_per_image"] = fin

    with tempfile.TemporaryDirectory() as d:
        td, pd = os.path.join(d, "true"), os.path.join(d, "pred")
        os.makedirs(td)
        os.makedirs(pd)
        for i in range(conse.shape[0]):
            sio.savemat(os.path.join(td, "img_%02d.mat" % i), {"inst_map": conse[i]})
            sio.savemat(os.path.join(pd, "img_%02d.mat" % i), {"inst_map": _pred_of(conse[i], i)})
        compute_stats.run_nuclei_inst_stat(pd, td)  # warm
        t1 = time.perf_counter()
        metrics = compute_stats.run_nuclei_inst_stat(pd, td)
        res["run_nuclei_inst_stat_s_per_image"] = (time.perf_counter() - t1) / conse.shape[0]
        res["run_nuclei_inst_stat_mean"] = np.mean(metrics, axis=-1).tolist()
    with open(os.path.join(args.out, "bench_stats.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))
    ok = all(res[k]["table_equals_oracle"] for k in ("14x1000x1000", "1x4096x4096"))
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
