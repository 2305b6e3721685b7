"""Benchmark of the per-nucleus measurements (hvn_inst_features) on the H100.

    python tools/bench_features.py --out DIR [--reps 20] [--repeats 3] [--batch 32]

Reports, as JSON in DIR/h100_bench_features.json:
* the device time of one hvn_inst_features_dev call (CUDA events on the context stream around the whole call,
  including its argument check and status read-back) on 16 seeded 1000 x 1000 maps in one call and on one
  4096 x 4096 map (tools/bench_stats.py's generators), with a seeded RGB image and prediction map, and whether every
  row equals the float64 restatement (tests/features_ref.py; orientation within 4 ulp, np_prob_mean within 1e-12);
* for scale only, measured on the host CPU: the restatement's per-nucleus Python loop on the same 1000 x 1000 maps;
* tile mode (`process_file_list`, writers included) with and without `save_features` on tools/bench_tiles.py's
  workloads, the two arms alternated in one process (images/s, median and spread);
* the card name, power limit and max SM clock (nvidia-smi query) read in the same run.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import features_ref as F  # noqa: E402
from hover_net_b200 import synth  # noqa: E402
from hover_net_b200.models.hovernet.post_proc import _ctx  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def _table(inst):
    """Instance-table rows [n,10] (id, bbox, area) of every id of inst, ascending."""
    from scipy import ndimage
    objs = ndimage.find_objects(inst)
    area = np.bincount(inst.ravel(), minlength=len(objs) + 1)
    rows = [[i + 1, s[0].start, s[1].start, s[0].stop, s[1].stop, area[i + 1], 0, 0, 0, 0]
            for i, s in enumerate(objs) if s is not None]
    return np.array(rows, dtype=np.int64).reshape(-1, 10)


def _contours(ctx, inst, table):
    """The device contours (hvn_contours_dev) of the rows of table: (pts [m,2], offs [n+1])."""
    H, W = inst.shape
    n = len(table)
    cap = max(4096, H * W // 4)
    host = [np.ascontiguousarray(inst), np.ascontiguousarray(table), np.array([n], np.int32)]
    d = [ctx.malloc(a.nbytes) for a in host] + [ctx.malloc(cap * 8), ctx.malloc((n + 1) * 4)]
    try:
        for dp, a in zip(d, host):
            ctx.h2d(dp, a, a.nbytes)
        ctx.contours_dev(d[0], d[1], d[2], 1, H, W, n, d[3], cap, d[4])
        offs = np.empty(n + 1, np.int32)
        ctx.d2h(offs, d[4], offs.nbytes)
        ctx.sync()
        assert offs[-1] <= cap
        pts = np.empty((int(offs[-1]), 2), np.int32)
        ctx.d2h(pts, d[3], pts.nbytes)
        ctx.sync()
        return pts, offs
    finally:
        for dp in d:
            ctx.free(dp)


def _group(maps, seed):
    ctx = _ctx()
    tables, ptsl, offs, ro, imgs, preds = [], [], [0], [0], [], []
    rng = np.random.default_rng(seed)
    for m in maps:
        t = _table(m)
        p, o = _contours(ctx, m, t)
        tables.append(t)
        ptsl.append(p)
        offs.extend((o[1:] + offs[-1]).tolist())
        ro.append(ro[-1] + len(t))
        imgs.append(rng.integers(0, 256, m.shape + (3,), dtype=np.uint8))
        preds.append(rng.uniform(0, 1, m.shape + (4,)).astype(np.float32))
    return (np.concatenate(tables), np.concatenate(ptsl), np.array(offs, np.int32), np.array(ro, np.int32), imgs,
            preds)


def _time_dev(maps, reps, seed, check_rows):
    ctx = _ctx()
    table, pts, offs, ro, imgs, preds = _group(maps, seed)
    cat = lambda arrs: np.ascontiguousarray(np.concatenate([a.reshape(-1) for a in arrs]))  # noqa: E731
    host = [cat(maps).astype(np.int32), cat(imgs), cat(preds), table, ro, pts, offs]
    n = len(table)
    d = [ctx.malloc(max(1, a.nbytes)) for a in host]
    d_f = ctx.malloc(n * 18 * 8)
    shapes = np.array([m.shape for m in maps], np.int32)
    try:
        for dp, a in zip(d, host):
            ctx.h2d(dp, a, a.nbytes)

        def call():
            ctx.inst_features_dev(len(maps), shapes, d[0], d[1], d[2], 4, d[3], d[4], n, d[5], d[6], d_f)
        for _ in range(3):
            call()
        ms = []
        for _ in range(reps):
            ctx.timer_start()
            call()
            ms.append(ctx.timer_stop())
        feats = np.empty((n, 18), np.float64)
        ctx.d2h(feats, d_f, feats.nbytes)
        ctx.sync()
    finally:
        for dp in d + [d_f]:
            ctx.free(dp)
    # the restatement on every row (check_rows None) or on a seeded sample of rows
    rows = np.arange(n) if check_rows is None else np.random.default_rng(seed).choice(n, min(n, check_rows), False)
    mapk = np.searchsorted(ro, rows, side="right") - 1
    ok = True
    t0 = time.perf_counter()
    for r, k in zip(rows, mapk):
        want = F.row_features(maps[k], table[r], pts[offs[r]:offs[r + 1]], imgs[k], preds[k][..., 1])
        got = feats[r]
        ex = [c for c in range(17) if c != 9]
        ok = ok and np.array_equal(got[ex].view(np.int64), want[ex].view(np.int64))
        ok = ok and abs(int(got[9:10].view(np.int64)[0]) - int(want[9:10].view(np.int64)[0])) <= 4
        ok = ok and abs(got[17] - want[17]) <= 1e-12 * abs(want[17])
    host_s = time.perf_counter() - t0
    px = sum(m.size for m in maps)
    bbox_px = int(((table[:, 3] - table[:, 1]) * (table[:, 4] - table[:, 2])).sum())
    return {"maps": len(maps), "pixels": px, "rows": n, "contour_points": int(offs[-1]), "bbox_pixels": bbox_px,
            "call_ms_median": float(np.median(ms)), "call_ms_min": float(np.min(ms)),
            "call_ms_max": float(np.max(ms)), "rows_checked": int(len(rows)), "equals_restatement": bool(ok),
            "host_restatement_s_per_nucleus": host_s / max(1, len(rows))}


def _tile_arms(name, w, repeats, batch):
    import cv2
    from bench_tiles import _image
    from hover_net_b200.infer.tile import InferManager
    d = tempfile.mkdtemp(prefix="bench_features_")
    os.makedirs(d + "/in")
    for i in range(w["n"]):
        cv2.imwrite("%s/in/%04d.png" % (d, i), cv2.cvtColor(_image(w["size"], 500 + i), cv2.COLOR_RGB2BGR))
    mgr = InferManager(method={"model_args": {"nr_types": w["nt"], "mode": w["mode"]},
                               "model_path": synth.make_state_dict(w["mode"], w["nt"], seed=0)}, type_info_path=None)
    run_args = {"batch_size": batch, "patch_input_shape": w["win"], "patch_output_shape": w["msk"],
                "input_dir": d + "/in", "mem_usage": 0.2}
    arms = {"tile": lambda: mgr.process_file_list(dict(run_args, output_dir=d + "/off")),
            "tile_save_features": lambda: mgr.process_file_list(dict(run_args, output_dir=d + "/on",
                                                                     save_features=True))}
    for f in arms.values():
        f()
    t = {k: [] for k in arms}
    for _ in range(repeats):
        for k, f in arms.items():
            t0 = time.perf_counter()
            f()
            t[k].append(time.perf_counter() - t0)
    res = {"workload": name, **w, "batch": batch, "repeats": repeats}
    for k, v in t.items():
        ips = sorted(w["n"] / x for x in v)
        res[k] = {"images_per_s_median": float(np.median(ips)), "images_per_s_min": ips[0],
                  "images_per_s_max": ips[-1]}
    mgr.net.ctx.close()
    shutil.rmtree(d, ignore_errors=True)
    return res


def main():
    from bench_tiles import WORKLOADS
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    res = {"card": _card()}
    conse = [synth.tiled_instances(1000, 1000, block=250, seed=s, n_unique=8) for s in range(16)]
    big = [synth.tiled_instances(4096, 4096, seed=99)]
    res["16x1000x1000"] = _time_dev(conse, a.reps, 1, None)
    print(json.dumps(res["16x1000x1000"]), flush=True)
    res["1x4096x4096"] = _time_dev(big, a.reps, 2, 2000)
    print(json.dumps(res["1x4096x4096"]), flush=True)
    res["host_restatement_note"] = ("host_restatement_s_per_nucleus: tests/features_ref.py's per-nucleus Python loop, "
                                    "measured on the host CPU of the GPU machine, for scale only")
    res["tile_mode"] = []
    for name, w in WORKLOADS.items():
        r = _tile_arms(name, w, a.repeats, a.batch)
        print(json.dumps(r), flush=True)
        res["tile_mode"].append(r)
    res["card_after"] = _card()
    with open(os.path.join(a.out, "h100_bench_features.json"), "w") as f:
        json.dump(res, f, indent=1)
    ok = res["16x1000x1000"]["equals_restatement"] and res["1x4096x4096"]["equals_restatement"]
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
