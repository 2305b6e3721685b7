"""Benchmark of the validation loss (hvn_valid_loss_dev) against the validation step without it (hvn_valid_dev) on one
GPU.

Workload: 128 original-mode 270 x 270 patches (the validation geometry of the reference's original mode; output crop
80 x 80), nr_types 5, seeded weights and instance maps.  In one process:
* hvn_valid_loss_dev and hvn_valid_dev alternated, --reps calls each after a warm-up, host clock around calls that
  end in a stream synchronise: seconds per call and the time ratio;
* then, in a separate loop with option "profile" = 1, the loss reduction's own CUDA-event time (hvn_stage_ms
  "loss": k_loss_reduce + k_loss_final) and the bytes it must move, computed from the shapes: per output pixel the
  (4 + nr_types) fp32 probabilities, the fp32 HV target pair and the int32 instance and type labels, plus the
  per-block partials written and read once;
* the counts of both calls compared, and the card name, power limit and max SM clock (nvidia-smi) read in the same
  run.

usage: python tools/bench_loss.py --out DIR [--reps N] [--batch B]
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


def loss_bytes(B, h, w, nt):
    ns = 10 + (1 + 3 * nt if nt else 0)
    tiles = B * -(-h // 32) * -(-w // 32)
    per_px = (4 + nt) * 4 + 8 + 4 + (4 if nt else 0)
    return B * h * w * per_px + 2 * tiles * ns * 8


def bench(reps, B):
    from hover_net_b200.models.hovernet.net_desc import create_model
    mode, nt, H = "original", 5, 270
    net = create_model(mode=mode, nr_types=nt)
    net.load_state_dict(synth.make_state_dict(mode, nt, seed=0), strict=True)
    ctx = net.ctx
    imgs = synth.make_patches(B, H, seed=7)
    inst = np.stack([synth.synth_instances(H, H, seed=200 + i % 16) for i in range(B)]).astype(np.int32)
    typ = np.where(inst > 0, inst % nt, 0).astype(np.int32)
    oh, ow, _ = ctx.out_shape(H, H)
    nc, ns = 3 + 2 * nt, 11 + 3 * nt
    bufs = [ctx.malloc(n) for n in (imgs.nbytes, inst.nbytes, typ.nbytes, nc * 8, 8, B * 4, ns * 8, nc * 8, 8)]
    d_img, d_inst, d_typ, d_cnt, d_sse, d_fl, d_sums, d_cnt2, d_sse2 = bufs
    t = {"valid": [], "valid_loss": []}
    try:
        ctx.h2d(d_img, imgs, imgs.nbytes)
        ctx.h2d(d_inst, inst, inst.nbytes)
        ctx.h2d(d_typ, typ, typ.nbytes)
        run = {"valid": lambda: ctx.valid_dev(d_img, d_inst, d_typ, B, H, H, d_cnt, d_sse, d_fl),
               "valid_loss": lambda: ctx.valid_loss_dev(d_img, d_inst, d_typ, B, H, H, d_cnt2, d_sse2, d_fl,
                                                        d_sums)}
        for f in run.values():  # warm-up: plans, arenas, module load
            f()
            f()
        for _ in range(reps):
            for name, f in run.items():
                t0 = time.perf_counter()
                f()  # both end in a stream synchronise
                t[name].append(time.perf_counter() - t0)
        c1, c2 = np.zeros(nc, np.int64), np.zeros(nc, np.int64)
        ctx.d2h(c1, d_cnt, nc * 8)
        ctx.d2h(c2, d_cnt2, nc * 8)
        sums = np.zeros(ns)
        ctx.d2h(sums, d_sums, ns * 8)
        ctx.set_option("profile", 1)
        kms = []
        for _ in range(reps):
            run["valid_loss"]()
            kms.append(ctx.stage_ms("loss"))
        ctx.set_option("profile", 0)
    finally:
        for p in bufs:
            ctx.free(p)
        ctx.close()
    from hover_net_b200.models.hovernet import run_desc
    res = {"mode": mode, "nr_types": nt, "batch": B, "patch": H, "crop": [oh, ow], "reps": reps,
           "counts_equal": bool(np.array_equal(c1, c2)),
           "loss_scalars_last": run_desc.loss_scalars(sums, B * oh * ow)}
    for name, v in t.items():
        med = float(np.median(v))
        res[name] = {"s_median": med, "s_min": float(min(v)), "s_max": float(max(v)), "patches_per_s": B / med}
    res["valid_loss_over_valid_time"] = res["valid_loss"]["s_median"] / res["valid"]["s_median"]
    kmed = float(np.median(kms))
    nbytes = loss_bytes(B, oh, ow, nt)
    res["loss_kernels"] = {"ms_median": kmed, "ms_min": float(min(kms)), "ms_max": float(max(kms)),
                           "bytes": nbytes, "GB_per_s": nbytes / (kmed * 1e-3) / 1e9,
                           "share_of_valid_call": kmed * 1e-3 / res["valid"]["s_median"]}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--batch", type=int, default=128)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    res = {"card": _card(), "loss": bench(args.reps, args.batch)}
    with open(os.path.join(args.out, "bench_loss.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))
    sys.exit(0 if res["loss"]["counts_equal"] else 1)


if __name__ == "__main__":
    main()
