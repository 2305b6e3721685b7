"""Benchmark of the two convolution precisions ("highest", "high") on the H100, in one process.

    python tools/bench_precision.py --out DIR [--repeats 4] [--steps 5] [--warmup 2]

Workload: BASELINE configs[2], the one `bench.py` runs by default -- 256 synthetic `original`-mode 270x270 patches,
nr_types 5, the same synthetic checkpoint (synth.make_state_dict seed 0) and the same patches (bench.make_batch seed 1).
A step is forward + instance post-processing on device buffers (hvn_forward_postproc_dev), as bench.py's timed step.
Both precisions get a context of their own; the timed windows alternate between them (order flipped every repeat) so
that clock drift and neighbours on the host hit both alike.  Reports, as JSON in DIR/bench_precision.json, per
precision:
* tiles/s: patches over the summed device time of the timed steps (CUDA events on the library stream around each step;
  an L2 flush runs between steps, outside the events), median and spread over the repeats;
* conv_tc algorithmic TFLOP/s from a separate profile pass (option "profile" = 2: per-launch events, decoder branches
  serialised) and its share of the 989 TFLOP/s dense FP16 data-sheet figure.  The algorithmic FLOPs are the reference
  graph's 2*MACs; "highest" issues three tensor-core products per MAC (its ceiling is 1/3 of that figure), "high" one;
* plan_bytes: device bytes of the activation buffers of the plan the forward ran;
* max / mean abs error of the NP probability and the HV maps against the fp64 oracle on the first few patches;
and the card name, power limit and max SM clock (nvidia-smi query) read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP16_DENSE_TFLOPS = 989.0  # H100 SXM data sheet, dense FP16 / BF16
PRECISIONS = ("highest", "high")


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--repeats", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--oracle_patches", type=int, default=2)
    args = ap.parse_args()

    import torch
    from bench import make_batch
    from hover_net_b200 import synth
    from hover_net_b200.models.hovernet.net_desc import create_model
    from oracle import hovernet_torch as O

    if not torch.cuda.is_available():
        raise SystemExit("bench_precision: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    card = _card()
    dev = torch.device("cuda", 0)
    mode, nt, B, S = "original", 5, args.batch, 270
    sd = synth.make_state_dict(mode, nt, seed=0)
    nets = {}
    for p in PRECISIONS:
        nets[p] = create_model(mode=mode, input_ch=3, nr_types=nt, device=0, precision=p)
        nets[p].load_state_dict(sd, strict=True)
    ctx0 = nets["highest"].ctx
    oh, ow, oc = ctx0.out_shape(S, S)
    max_rows = max(16, oh * ow // 64)
    x = make_batch(B, S, seed=1)
    d_img = torch.from_numpy(x).to(dev)
    d_pred = torch.empty((B, oh, ow, oc), dtype=torch.float32, device=dev)
    d_inst = torch.empty((B, oh, ow), dtype=torch.int32, device=dev)
    d_tab = torch.zeros((B, max_rows, 10), dtype=torch.int64, device=dev)
    d_nr = torch.zeros((B,), dtype=torch.int32, device=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()

    def step(ctx):
        ctx.forward_postproc_dev(d_img.data_ptr(), B, S, S, d_pred.data_ptr(), d_inst.data_ptr(), d_tab.data_ptr(),
                                 max_rows, d_nr.data_ptr())

    for p in PRECISIONS:
        for _ in range(args.warmup):
            step(nets[p].ctx)
        nets[p].ctx.sync()
    torch.cuda.synchronize()

    tiles_s = {p: [] for p in PRECISIONS}
    for r in range(args.repeats):
        for p in (PRECISIONS if r % 2 == 0 else PRECISIONS[::-1]):
            ctx = nets[p].ctx
            ms = 0.0
            for _ in range(args.steps):
                flush.fill_(1)
                torch.cuda.synchronize()
                ctx.timer_start()
                step(ctx)
                ms += ctx.timer_stop()
            tiles_s[p].append(B * args.steps / (ms / 1e3))

    res = {}
    for p in PRECISIONS:
        ctx = nets[p].ctx
        plan_bytes = ctx.counter("plan_bytes")
        ctx.set_option("branch_streams", 0)  # per-launch event times must not overlap
        ctx.set_option("profile", 2)
        for _ in range(2):
            step(ctx)
        ctx.sync()
        tc_ms = ctx.stage_ms("conv_tc")
        tc_gflop = ctx.counter("flops:conv_tc") / 1e9
        cnn_ms = ctx.stage_ms("cnn")
        ctx.set_option("profile", 0)
        ctx.set_option("branch_streams", 1)
        tflops = tc_gflop / tc_ms if tc_ms > 0 else 0.0  # GFLOP / ms = TFLOP/s
        v = np.array(tiles_s[p])
        res[p] = {"tiles_per_s": float(np.median(v)), "tiles_per_s_repeats": [float(t) for t in v],
                  "spread": float((v.max() - v.min()) / np.median(v)),
                  "conv_tc": {"ms": tc_ms, "gflop": tc_gflop, "tflops_algorithmic": tflops,
                              "share_of_989": tflops / FP16_DENSE_TFLOPS,
                              "ceiling_share": 1.0 / 3.0 if p == "highest" else 1.0,
                              "launches": ctx.counter("launches:conv_tc")},
                  "cnn_ms_profiled": cnn_ms, "plan_bytes": int(plan_bytes)}

    # accuracy against the fp64 oracle on the first patches (same weights)
    n = args.oracle_patches
    ref = O.infer_step(x[:n], O.to_torch_state_dict(sd), mode, nt, dtype=torch.float64, device="cuda")
    for p in PRECISIONS:
        out = nets[p].ctx.forward(x[:n])
        e_np = np.abs(out[..., -3] - ref[..., -3])
        e_hv = np.abs(out[..., -2:] - ref[..., -2:])
        res[p]["error_vs_fp64"] = {"patches": n, "np_max": float(e_np.max()), "np_mean": float(e_np.mean()),
                                   "hv_max": float(e_hv.max()), "hv_mean": float(e_hv.mean()),
                                   "tp_mismatch": float((out[..., 0] != ref[..., 0]).mean())}
    for p in PRECISIONS:
        nets[p].ctx.close()

    summary = {"card": card, "workload": "BASELINE configs[2]: %d synthetic original-mode 270x270 patches, nr_types 5, "
                                        "forward + post-processing per step" % B,
               "repeats": args.repeats, "steps": args.steps, "warmup": args.warmup, "results": res,
               "speedup_high_over_highest": res["high"]["tiles_per_s"] / res["highest"]["tiles_per_s"]}
    with open(os.path.join(args.out, "bench_precision.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
