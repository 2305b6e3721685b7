"""Benchmark of test-time augmentation (option "tta") on the H100: plain vs TTA for both precisions, in one process.

    python tools/bench_tta.py --out DIR [--repeats 4] [--steps 3] [--warmup 1]

Workload: BASELINE configs[2], as tools/bench_precision.py -- 256 synthetic `original`-mode 270x270 patches, nr_types 5,
the synthetic checkpoint of synth.make_state_dict seed 0 and the patches of bench.make_batch seed 1.  A step is forward
+ instance post-processing on device buffers (hvn_forward_postproc_dev); under TTA the forward runs the 8 views of every
patch.  Per precision the two arms get a context each, and their timed windows alternate (order flipped every repeat);
the precisions run one after the other so that only two contexts' buffers are resident at a time.  Reports, as JSON in
DIR/bench_tta.json, per precision:
* input patches/s of each arm: patches over the summed device time of the timed steps (CUDA events on the library
  stream; an L2 flush runs between steps, outside the events), median and spread over the repeats;
* ratio = TTA patches/s / (plain patches/s / 8): 1 means TTA costs exactly its eight forwards;
* the device time of k_tta_views + k_tta_merge (profile pass, option "profile" = 2: per-launch events, decoder branches
  serialised), their share of that pass's forward time, and their bytes/s against the 3.35 TB/s HBM3 data-sheet figure.
  Bytes are the algorithmic ones: per input pixel 3 read + 8 x 3 written by the views; per output pixel 8 views x
  (nr_types + 3) fp32 read + 4 fp32 written by the merge;
* NP / HV max abs error of the TTA output against a TTA over the fp64 oracle network on the first few patches;
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
sys.path.insert(0, os.path.join(ROOT, "tests"))  # tta_ref: the host restatement of the views and the merge

HBM_TBPS = 3.35  # H100 SXM data sheet, HBM3
PRECISIONS = ("highest", "high")
ARMS = ("plain", "tta")


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--repeats", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--oracle_patches", type=int, default=2)
    args = ap.parse_args()

    import torch
    import tta_ref
    from bench import make_batch
    from hover_net_b200 import synth
    from hover_net_b200.models.hovernet.net_desc import create_model

    if not torch.cuda.is_available():
        raise SystemExit("bench_tta: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    card = _card()
    dev = torch.device("cuda", 0)
    mode, nt, B, S = "original", 5, args.batch, 270
    sd = synth.make_state_dict(mode, nt, seed=0)
    x = make_batch(B, S, seed=1)
    d_img = torch.from_numpy(x).to(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    n = args.oracle_patches
    ref = tta_ref.oracle_tta(x[:n], sd, mode, nt)

    res = {}
    for p in PRECISIONS:
        nets = {a: create_model(mode=mode, input_ch=3, nr_types=nt, device=0, precision=p, tta=(a == "tta"))
                for a in ARMS}
        for a in ARMS:
            nets[a].load_state_dict(sd, strict=True)
        oh, ow, oc = nets["plain"].ctx.out_shape(S, S)
        max_rows = max(16, oh * ow // 64)
        d_pred = torch.empty((B, oh, ow, oc), dtype=torch.float32, device=dev)
        d_inst = torch.empty((B, oh, ow), dtype=torch.int32, device=dev)
        d_tab = torch.zeros((B, max_rows, 10), dtype=torch.int64, device=dev)
        d_nr = torch.zeros((B,), dtype=torch.int32, device=dev)
        torch.cuda.synchronize()

        def step(ctx):
            ctx.forward_postproc_dev(d_img.data_ptr(), B, S, S, d_pred.data_ptr(), d_inst.data_ptr(), d_tab.data_ptr(),
                                     max_rows, d_nr.data_ptr())

        for a in ARMS:
            for _ in range(args.warmup):
                step(nets[a].ctx)
            nets[a].ctx.sync()
        torch.cuda.synchronize()

        rate = {a: [] for a in ARMS}
        for r in range(args.repeats):
            for a in (ARMS if r % 2 == 0 else ARMS[::-1]):
                ctx = nets[a].ctx
                ms = 0.0
                for _ in range(args.steps):
                    flush.fill_(1)
                    torch.cuda.synchronize()
                    ctx.timer_start()
                    step(ctx)
                    ms += ctx.timer_stop()
                rate[a].append(B * args.steps / (ms / 1e3))

        out = {}
        for a in ARMS:
            v = np.array(rate[a])
            out[a] = {"patches_per_s": float(np.median(v)), "patches_per_s_repeats": [float(t) for t in v],
                      "spread": float((v.max() - v.min()) / np.median(v)),
                      "plan_bytes": int(nets[a].ctx.counter("plan_bytes"))}
        out["ratio_tta_over_plain_div_8"] = out["tta"]["patches_per_s"] / (out["plain"]["patches_per_s"] / 8.0)

        ctx = nets["tta"].ctx  # profile pass: per-launch events, branches serialised
        ctx.set_option("branch_streams", 0)
        ctx.set_option("profile", 2)
        step(ctx)
        ctx.sync()
        tta_ms, cnn_ms = ctx.stage_ms("tta"), ctx.stage_ms("cnn")
        launches = ctx.counter("launches:tta")
        ctx.set_option("profile", 0)
        ctx.set_option("branch_streams", 1)
        nbytes = B * S * S * (3 + 8 * 3) + B * oh * ow * (8 * (nt + 3) + oc) * 4
        out["tta_kernels"] = {"ms": tta_ms, "launches": launches, "forward_ms_profiled": cnn_ms,
                              "share_of_forward": tta_ms / cnn_ms if cnn_ms > 0 else None, "bytes": nbytes,
                              "tb_per_s": nbytes / (tta_ms / 1e3) / 1e12 if tta_ms > 0 else None,
                              "share_of_3.35_tbps": nbytes / (tta_ms / 1e3) / 1e12 / HBM_TBPS if tta_ms > 0 else None}

        got = nets["tta"].ctx.forward(x[:n])
        out["tta_error_vs_fp64_oracle_tta"] = {
            "patches": n, "np_max": float(np.abs(got[..., -3] - ref[..., -3]).max()),
            "hv_max": float(np.abs(got[..., -2:] - ref[..., -2:]).max()),
            "hv_scale": float(np.abs(ref[..., -2:]).max()),
            "tp_mismatch": float((got[..., 0] != ref[..., 0]).mean())}
        for a in ARMS:
            nets[a].ctx.close()
        del d_pred, d_inst, d_tab, d_nr
        torch.cuda.empty_cache()
        res[p] = out

    summary = {"card": card, "workload": "BASELINE configs[2]: %d synthetic original-mode 270x270 patches, nr_types 5, "
                                        "forward + post-processing per step" % B,
               "repeats": args.repeats, "steps": args.steps, "warmup": args.warmup, "results": res}
    with open(os.path.join(args.out, "bench_tta.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
