"""Benchmark of the training targets and the fused validation step on one GPU.

* hvn_targets_dev on 256 instance maps of 270 x 270 (crop 80, seeded `synth_instances` maps, the original-mode
  validation geometry): CUDA-event time per call over --reps calls, after a warm-up; a few maps are checked against
  the numpy oracle first.
* hvn_valid_dev (forward + targets + counts) against hvn_forward_dev alone on the same batch of original-mode
  270 x 270 patches (nr_types 5, seeded weights), alternated in one process, --reps calls each: patches/s.
* the card name, power limit and max SM clock (nvidia-smi query) read in the same run.

usage: python tools/bench_valid.py --out DIR [--reps N] [--batch B]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hover_net_b200 import synth  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def bench_targets(reps):
    from hover_net_b200 import _lib
    from oracle import targets_oracle as O
    n, H, crop = 256, 270, 80
    uniq = [synth.synth_instances(H, H, seed=100 + k) for k in range(16)]
    maps = np.ascontiguousarray(np.stack([uniq[k % 16] for k in range(n)]), dtype=np.int32)
    ctx = _lib.Context(0)
    d_in, d_hv, d_fl = ctx.malloc(maps.nbytes), ctx.malloc(maps.nbytes * 2), ctx.malloc(n * 4)
    try:
        ctx.h2d(d_in, maps, maps.nbytes)
        ctx.targets_dev(d_in, n, H, H, crop, crop, d_hv, d_fl)
        hv = np.empty((n, H, H, 2), np.float32)
        ctx.d2h(hv, d_hv, hv.nbytes)
        same = all(hv[k].tobytes() == O.hv_map(maps[k], (crop, crop))[0].tobytes() for k in range(16))
        for _ in range(3):
            ctx.targets_dev(d_in, n, H, H, crop, crop, d_hv, d_fl)
        ms = []
        for _ in range(reps):
            ctx.timer_start()
            ctx.targets_dev(d_in, n, H, H, crop, crop, d_hv, d_fl)
            ms.append(ctx.timer_stop())
    finally:
        for p in (d_in, d_hv, d_fl):
            ctx.free(p)
        ctx.close()
    med = float(np.median(ms))
    return {"maps": n, "size": H, "crop": crop, "instances_per_map": float(np.mean([u.max() for u in uniq])),
            "ms_median": med, "ms_min": float(min(ms)), "ms_max": float(max(ms)), "maps_per_s": n / med * 1e3,
            "equals_oracle_16_maps": bool(same)}


def bench_valid(reps, B):
    from hover_net_b200.models.hovernet.net_desc import create_model
    mode, nt, H = "original", 5, 270
    net = create_model(mode=mode, nr_types=nt)
    net.load_state_dict(synth.make_state_dict(mode, nt, seed=0), strict=True)
    ctx = net.ctx
    imgs = synth.make_patches(B, H, seed=7)
    inst = np.stack([synth.synth_instances(H, H, seed=200 + i % 16) for i in range(B)]).astype(np.int32)
    typ = np.where(inst > 0, inst % nt, 0).astype(np.int32)
    oh, ow, oc = ctx.out_shape(H, H)
    nc = 3 + 2 * nt
    d_img, d_inst, d_typ = ctx.malloc(imgs.nbytes), ctx.malloc(inst.nbytes), ctx.malloc(typ.nbytes)
    d_out = ctx.malloc(B * oh * ow * oc * 4)
    d_cnt, d_sse, d_fl = ctx.malloc(nc * 8), ctx.malloc(8), ctx.malloc(B * 4)
    t = {"forward": [], "valid": []}
    try:
        ctx.h2d(d_img, imgs, imgs.nbytes)
        ctx.h2d(d_inst, inst, inst.nbytes)
        ctx.h2d(d_typ, typ, typ.nbytes)
        run = {"forward": lambda: (ctx.forward_dev(d_img, B, H, H, d_out), ctx.sync()),
               "valid": lambda: ctx.valid_dev(d_img, d_inst, d_typ, B, H, H, d_cnt, d_sse, d_fl)}
        for f in run.values():  # warm-up: plans, arenas, module load
            f()
            f()
        for _ in range(reps):
            for name, f in run.items():
                t0 = time.perf_counter()
                f()  # both end in a stream synchronise
                t[name].append(time.perf_counter() - t0)
        counts = np.zeros(nc, np.int64)
        ctx.d2h(counts, d_cnt, nc * 8)
    finally:
        for p in (d_img, d_inst, d_typ, d_out, d_cnt, d_sse, d_fl):
            ctx.free(p)
    res = {"mode": mode, "nr_types": nt, "batch": B, "reps": reps, "counts_last": counts.tolist()}
    for name, v in t.items():
        med = float(np.median(v))
        res[name] = {"s_median": med, "s_min": float(min(v)), "s_max": float(max(v)), "patches_per_s": B / med}
    res["valid_over_forward_time"] = res["valid"]["s_median"] / res["forward"]["s_median"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=128)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    res = {"card": _card()}
    res["targets"] = bench_targets(max(args.reps, 20))
    print("targets", json.dumps(res["targets"]))
    res["valid"] = bench_valid(args.reps, args.batch)
    print("valid", json.dumps(res["valid"]))
    with open(os.path.join(args.out, "bench_valid.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))
    sys.exit(0 if res["targets"]["equals_oracle_16_maps"] else 1)


if __name__ == "__main__":
    main()
