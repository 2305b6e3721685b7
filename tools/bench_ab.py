"""A/B benchmark of two source trees of this repository on one GPU: a base revision against the working tree.

    python tools/bench_ab.py prepare [--rev HEAD] [--dir ab_base]     # no GPU needed: export + build the base tree
    python tools/bench_ab.py run --out DIR [--base ab_base] [--rounds orig256=5,fast64=3,tile4k=3] [--steps 5] [--warmup 3]

`prepare` exports the base revision (`git archive`) into an untracked directory and builds it there with the same
`__graft_entry__.build()` as the working tree, so that both trees' native code exists before any GPU time is spent.

`run` runs `bench.py --gpus 1` from both trees in one process tree, alternating them (base first in even rounds, the
working tree first in odd ones) so that clock drift and neighbours on the host hit both alike.  It writes
DIR/bench_ab.json with, per workload, every round's `value` and `e2e.value` (the host-buffer entry point) for both
trees, their medians, their spread ((max - min) / median) and the ratios of the medians, and each tree's e2e
`h2d_bytes_per_step` / `d2h_bytes_per_step`; the card's name, power limit and max SM clock, read by nvidia-smi in
the same run; and whether both trees' `--dump-outputs` (written to a temporary directory, removed afterwards) are
bit-identical:
* orig256 and fast64 in precision "highest" (the dump of the first timed round: it is written after the timed steps);
* orig256 and fast64 in precision "high" (`--opt precision=1`, one extra short run per tree).
It also runs `tools/gpu_diag.py layers original 32` (per-layer device time, kernels serialised) in both trees and
writes the per-class tables of this tree's `tools/layer_classes.py` for both logs to DIR/layer_classes_ab.md.
bench.py itself runs unchanged; neither tree is written to (Python byte-code writing is off).
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _env():
    env = dict(os.environ)
    env["PYTHONDONTWRITEBYTECODE"] = "1"
    return env


def prepare(args):
    d = os.path.abspath(os.path.join(ROOT, args.dir))
    if os.path.exists(d):
        shutil.rmtree(d)
    os.makedirs(d)
    arc = subprocess.run(["git", "-C", ROOT, "archive", args.rev], check=True, capture_output=True).stdout
    subprocess.run(["tar", "-x", "-C", d], input=arc, check=True)
    subprocess.run([sys.executable, "-B", "-c", "import __graft_entry__ as g; g.build()"], cwd=d, check=True, env=_env())
    rev = subprocess.run(["git", "-C", ROOT, "rev-parse", args.rev], check=True, capture_output=True, text=True).stdout.strip()
    with open(os.path.join(d, "AB_REVISION"), "w") as f:
        f.write(rev + "\n")
    print("base tree %s at %s" % (rev, d))


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    if q.returncode != 0:
        raise SystemExit("bench_ab: nvidia-smi failed: " + q.stderr.strip())
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _bench(tree, workload, steps, warmup, extra=(), dump=None):
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
           "--workload", workload, "--no-cpu-baseline"] + list(extra)
    if dump:
        cmd += ["--dump-outputs", dump]
    p = subprocess.run(cmd, cwd=tree, capture_output=True, text=True, env=_env())
    lines = [l for l in p.stdout.splitlines() if l.startswith("{")]
    if p.returncode != 0 or not lines:
        raise SystemExit("bench_ab: %s in %s failed (%d):\n%s\n%s" % (" ".join(cmd), tree, p.returncode, p.stdout[-2000:], p.stderr[-4000:]))
    return json.loads(lines[-1])


def _same_dumps(a, b):
    """True when both directories hold the same .npy files with the same bytes (NaN payloads included)."""
    fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
    if fa != fb:
        return False, "files differ: %s vs %s" % (fa, fb)
    for f in fa:
        x, y = np.load(os.path.join(a, f)), np.load(os.path.join(b, f))
        if x.shape != y.shape or x.dtype != y.dtype or x.tobytes() != y.tobytes():
            n = int(np.sum(x != y)) if x.shape == y.shape else -1
            return False, "%s differs (%d elements)" % (f, n)
    return True, "%d files bit-identical" % len(fa)


def _stats(v):
    med = statistics.median(v)
    return {"values": v, "median": med, "spread": (max(v) - min(v)) / med}


def run(args):
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ab: no CUDA device")
    base = os.path.abspath(os.path.join(ROOT, args.base))
    if not os.path.isfile(os.path.join(base, "bench.py")):
        raise SystemExit("bench_ab: no base tree at %s (run `prepare` first)" % base)
    out = os.path.abspath(args.out)
    os.makedirs(out, exist_ok=True)
    trees = {"base": base, "this": ROOT}
    rev = open(os.path.join(base, "AB_REVISION")).read().strip() if os.path.exists(os.path.join(base, "AB_REVISION")) else None
    res = {"card": _card(), "base_revision": rev, "steps": args.steps, "warmup": args.warmup, "workloads": {}, "outputs": {}}
    dumps = tempfile.mkdtemp(prefix="bench_ab_")   # output dumps: compared here, then removed
    for spec in args.rounds.split(","):
        wl, n = spec.split("=")
        vals, e2e, copies = {"base": [], "this": []}, {"base": [], "this": []}, {}
        for r in range(int(n)):
            for t in (("base", "this") if r % 2 == 0 else ("this", "base")):
                dump = os.path.join(dumps, t, wl + "_highest") if r == 0 and wl in ("orig256", "fast64") else None
                line = _bench(trees[t], wl, args.steps, args.warmup, dump=dump)
                vals[t].append(line["value"])
                e2e[t].append(line["e2e"]["value"])
                copies[t] = {k: line["e2e"].get(k) for k in ("h2d_bytes_per_step", "d2h_bytes_per_step")}
                print("%s round %d %s: %.3f %s" % (wl, r, t, line["value"], line["unit"]), flush=True)
        w = {t: _stats(v) for t, v in vals.items()}
        w["ratio"] = w["this"]["median"] / w["base"]["median"]
        w["unit"] = line["unit"]
        w["e2e"] = {t: _stats(v) for t, v in e2e.items()}
        w["e2e"]["ratio"] = w["e2e"]["this"]["median"] / w["e2e"]["base"]["median"]
        w["e2e"]["copies"] = copies
        res["workloads"][wl] = w
        for tag, x in (("value", w), ("e2e", w["e2e"])):
            print("%s %s: this / base = %.4f (spread base %.2f %%, this %.2f %%)" % (
                wl, tag, x["ratio"], 100 * x["base"]["spread"], 100 * x["this"]["spread"]), flush=True)
    for wl in ("orig256", "fast64"):
        for t in ("base", "this"):
            _bench(trees[t], wl, 1, 1, extra=["--opt", "precision=1"], dump=os.path.join(dumps, t, wl + "_high"))
        for prec in ("highest", "high"):
            key = "%s_%s" % (wl, prec)
            a, b = os.path.join(dumps, "base", key), os.path.join(dumps, "this", key)
            if os.path.isdir(a) and os.path.isdir(b):
                same, why = _same_dumps(a, b)
                res["outputs"][key] = {"bit_identical": same, "detail": why}
                print("outputs %s: %s" % (key, why), flush=True)
    shutil.rmtree(dumps, ignore_errors=True)
    tables = []
    for t in ("base", "this"):
        log = os.path.join(out, "layers_original_32_%s.log" % t)
        p = subprocess.run([sys.executable, "tools/gpu_diag.py", "layers", "original", "32"], cwd=trees[t],
                           capture_output=True, text=True, env=_env())
        with open(log, "w") as f:
            f.write(p.stdout + p.stderr)
        if p.returncode != 0:
            raise SystemExit("bench_ab: gpu_diag layers failed in %s:\n%s" % (trees[t], p.stderr[-4000:]))
        q = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "layer_classes.py"), log], capture_output=True,
                           text=True, env=_env(), check=True)
        tables.append("### %s\n\n%s" % ("base " + (rev or "") if t == "base" else "this tree", q.stdout.replace(log, os.path.basename(log))))
    with open(os.path.join(out, "layer_classes_ab.md"), "w") as f:
        f.write("Card: %(name)s, power limit %(power_limit)s, max SM clock %(max_sm_clock)s\n\n" % res["card"] + "\n".join(tables))
    with open(os.path.join(out, "bench_ab.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: res[k] for k in ("card", "outputs")}))


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    p = sub.add_parser("prepare")
    p.add_argument("--rev", default="HEAD")
    p.add_argument("--dir", default="ab_base")
    r = sub.add_parser("run")
    r.add_argument("--out", required=True)
    r.add_argument("--base", default="ab_base")
    r.add_argument("--rounds", default="orig256=5,fast64=3,tile4k=3")
    r.add_argument("--steps", type=int, default=5)
    r.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    prepare(args) if args.cmd == "prepare" else run(args)


if __name__ == "__main__":
    main()
