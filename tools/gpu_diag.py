"""GPU-box diagnostics: per-stage timing and mismatch details (development aid)."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from hover_net_b200 import _lib, synth, arch
from oracle import postproc_oracle as P

def pp():
    c = _lib.Context(0)
    for (h, w, nt, n) in [(80, 80, None, 4), (164, 164, 6, 8), (270, 270, None, 2)]:
        maps = np.stack([synth.synth_pred_map(h, w, nt, s) for s in range(n)])
        t = time.time(); inst, table, nrows = c.postproc(maps, nt); dt = time.time() - t
        bad = 0
        for i in range(n):
            oi, ot = P.process_table(maps[i], nt)
            ok_i = np.array_equal(inst[i], oi); ok_t = int(nrows[i]) == len(ot) and np.array_equal(table[i, :len(ot)], ot)
            if not (ok_i and ok_t):
                bad += 1
                print("  MISMATCH map", i, "inst px diff", int((inst[i] != oi).sum()), "rows", int(nrows[i]), len(ot))
        print("pp %dx%d nt=%s n=%d: bad=%d wall=%.1fms" % (h, w, nt, n, bad, dt * 1e3))
    c.set_option("profile", 1)
    maps = np.stack([synth.synth_pred_map(164, 164, 6, s) for s in range(64)])
    for _ in range(3):
        c.postproc(maps, 6)
    print("pp 64x164^2 device ms:", c.stage_ms("postproc"))
    c.close()

def cnn():
    import torch
    from oracle import hovernet_torch as O
    from hover_net_b200.models.hovernet.net_desc import create_model
    for mode, nt in (("original", None), ("fast", 6)):
        g = np.load("tests/golden/cnn_%s_%s.npz" % (mode, nt))
        x = synth.make_patches(int(g["batch"]), arch.PATCH_GEOMETRY[mode][0], seed=7)
        net = create_model(mode=mode, nr_types=nt)
        net.load_state_dict(synth.make_state_dict(mode, nt, 0))
        for path in (1, 0):
            net.ctx.set_option("conv_path", path); net.ctx.set_option("profile", 1)
            out = net.ctx.forward(x)
            d = np.abs(out[..., -3:] - g["out"][..., -3:])
            print("cnn %s nt=%s path=%d: max err %.3e mean %.3e  finite=%s  ms=%.2f tc=%d" % (
                mode, nt, path, d.max(), d.mean(), np.isfinite(out).all(), net.ctx.stage_ms("cnn"), net.ctx.counter("tc_launches")))
            if nt: print("   tp mismatch frac", (out[..., 0] != g["out"][..., 0]).mean())
        net.ctx.close()

if __name__ == "__main__":
    what = sys.argv[1:] or ["pp", "cnn"]
    if "pp" in what: pp()
    if "cnn" in what: cnn()


def _knobs(net):
    """development knobs from the environment: HVN_TC_SEG=<64-channel slices per accumulation segment>"""
    if os.environ.get("HVN_TC_SEG"):
        net.ctx.set_option("tc_seg_chunks", int(os.environ["HVN_TC_SEG"]))


def tc(mode="fast", nt=6, verbose=False):
    """per-layer wgmma-vs-referee self test (conv_path=2), then the end-to-end check"""
    import re
    from hover_net_b200.models.hovernet.net_desc import create_model
    nt = {"fast": 6, "original": 5}[mode]
    g = np.load("tests/golden/cnn_%s_%s.npz" % (mode, nt))
    x = synth.make_patches(int(g["batch"]), arch.PATCH_GEOMETRY[mode][0], seed=7)
    net = create_model(mode=mode, nr_types=nt)
    net.load_state_dict(synth.make_state_dict(mode, nt, 0))
    _knobs(net)
    for seg in (4,):
        net.ctx.set_option("tc_seg_chunks", seg)
        net.ctx.set_option("conv_path", 2)
        out = net.ctx.forward(x)
        log = net.ctx.debug_log().strip().split("\n")
        rows = []
        for ln in log:
            m = re.findall(r"diff ([0-9.e+-]+) \(ref ([0-9.e+-]+)\)", ln)
            rel = max(float(d) / max(float(r), 1e-30) for d, r in m if float(r) > 0) if m else 0
            rows.append((rel, ln))
        rows.sort(reverse=True)
        if verbose:
            print("\n".join(log))
        halo_rows = [r for r in rows if "H bn=" in r[1]]
        print("seg=%d: %d layers, %d on the halo variant (worst halo rel %.2e); worst layers by relative diff:" % (
            seg, len(rows), len(halo_rows), max([r[0] for r in halo_rows] or [0.0])))
        for rel, ln in rows[:4]:
            print("   rel %.2e | %s" % (rel, ln[:150]))
        d = np.abs(out[..., -3:] - g["out"][..., -3:])
        print("seg=%d tc e2e %s: max err %.3e mean %.3e finite=%s tc_launches=%d" % (seg, mode, d.max(), d.mean(), np.isfinite(out).all(), net.ctx.counter("tc_launches")))
        net.ctx.set_option("conv_path", 0); net.ctx.set_option("profile", 2)
        for _ in range(2):
            out = net.ctx.forward(x)
        for cls in ("conv_tc", "conv_ref", "conv0", "bnrelu", "head"):
            ms = net.ctx.stage_ms(cls); fl = net.ctx.counter("flops:" + cls); n = net.ctx.counter("launches:" + cls)
            print("  %-8s %8.3f ms  %4d launches  %8.1f GFLOP  %7.1f TFLOP/s" % (cls, ms, n, fl / 1e9, fl / 1e9 / max(ms, 1e-9)))
        print("  cnn total ms", net.ctx.stage_ms("cnn"), "batch", x.shape[0])
        net.ctx.set_option("profile", 0)
    net.ctx.close()


if __name__ == "__main__" and "tc" in sys.argv[1:]:
    tc(*(sys.argv[sys.argv.index("tc") + 1:sys.argv.index("tc") + 2] or ["fast"]), verbose="v" in sys.argv)


def layers(mode="fast", B=8):
    """per-layer device time at batch B (profile=3)"""
    from hover_net_b200.models.hovernet.net_desc import create_model
    nt = {"fast": 6, "original": 5}[mode]
    x = synth.make_patches(B, arch.PATCH_GEOMETRY[mode][0], seed=7)
    net = create_model(mode=mode, nr_types=nt)
    net.load_state_dict(synth.make_state_dict(mode, nt, 0))
    _knobs(net)
    net.ctx.set_option("chunk", B)
    net.ctx.set_option("branch_streams", 0)
    net.ctx.forward(x)
    net.ctx.set_option("profile", 3)
    net.ctx.forward(x)
    print(net.ctx.debug_log())
    for cls in ("conv_tc", "conv_ref", "conv0", "bnrelu", "head"):
        ms = net.ctx.stage_ms(cls); fl = net.ctx.counter("flops:" + cls); n = net.ctx.counter("launches:" + cls)
        print("  %-8s %8.3f ms  %4d launches  %8.1f GFLOP  %7.1f TFLOP/s" % (cls, ms, n, fl / 1e9, fl / 1e9 / max(ms, 1e-9)))
    print("  cnn total ms", net.ctx.stage_ms("cnn"), "batch", B)
    net.ctx.close()


if __name__ == "__main__" and "layers" in sys.argv[1:]:
    i = sys.argv.index("layers")
    layers(sys.argv[i + 1] if len(sys.argv) > i + 1 else "fast", int(sys.argv[i + 2]) if len(sys.argv) > i + 2 else 8)


def cpuf():
    """torch CPU forward time vs thread count (to pick a fair reference-arm setting)"""
    import torch
    from oracle import hovernet_torch as O
    sd = O.to_torch_state_dict(synth.make_state_dict("fast", 6, 0))
    x = synth.make_patches(4, 256, seed=1)
    for th in (8, 16, 32, 64, 128):
        torch.set_num_threads(th)
        O.infer_step(x[:1], sd, "fast", 6)
        t = time.time(); O.infer_step(x, sd, "fast", 6); dt = time.time() - t
        print("torch cpu threads=%d: %.3f s/patch (batch 4)" % (th, dt / 4))


if __name__ == "__main__" and "cpuf" in sys.argv[1:]:
    cpuf()


def ppprof(B=64):
    """per-kernel post-processing time on CNN-output maps and on synthetic nuclei maps"""
    from hover_net_b200.models.hovernet.net_desc import create_model
    net = create_model(mode="fast", nr_types=6)
    net.load_state_dict(synth.make_state_dict("fast", 6, 0))
    x = synth.make_patches(8, 256, seed=1)
    x = np.concatenate([x] * (B // 8))
    pred = net.ctx.forward(x)
    fg = (pred[..., 1] >= 0.5)
    print("CNN-output maps: fg fraction %.3f" % fg.mean())
    net.ctx.set_option("profile", 3)
    for name, maps in (("cnn-output", pred), ("synthetic nuclei", np.stack([synth.synth_pred_map(164, 164, 6, s) for s in range(B)]))):
        net.ctx.postproc(maps, 6); net.ctx.postproc(maps, 6)
        print("== %s: total %.3f ms for %d maps" % (name, net.ctx.stage_ms("postproc"), B))
        rows = [l for l in net.ctx.debug_log().split("\n") if l.startswith("pp ") and "stats" not in l]
        rows.sort(key=lambda l: -float(l.split()[-2]))
        print("\n".join(rows[:8]))
        print("\n".join(l for l in net.ctx.debug_log().split("\n") if "pp stats" in l))
    net.ctx.close()


if __name__ == "__main__" and "ppprof" in sys.argv[1:]:
    ppprof()


def sweep():
    """CNN-only device time vs chunk size and branch streams (B=64, fast)"""
    from hover_net_b200.models.hovernet.net_desc import create_model
    net = create_model(mode="fast", nr_types=6)
    net.load_state_dict(synth.make_state_dict("fast", 6, 0))
    x = np.concatenate([synth.make_patches(8, 256, seed=1)] * 8)
    net.ctx.set_option("profile", 1)
    ref = None
    for bs in (0, 1):
        for chunk in (8, 16, 32):
            net.ctx.set_option("branch_streams", bs); net.ctx.set_option("chunk", chunk)
            out = net.ctx.forward(x); out = net.ctx.forward(x)
            if ref is None: ref = out
            print("branch_streams=%d chunk=%2d: cnn %.2f ms for 64 patches (%.3f ms/patch) same=%s" % (
                bs, chunk, net.ctx.stage_ms("cnn"), net.ctx.stage_ms("cnn") / 64, np.array_equal(out, ref)))
    net.ctx.close()


if __name__ == "__main__" and "sweep" in sys.argv[1:]:
    sweep()


def ab(mode="original", B=16, configs=("base:",), reps=5):
    """A/B per-layer device times inside ONE process: the configurations (launch-time knobs, "tag:key=value,...") are
    interleaved `reps` times and the per-layer MEDIAN is reported, so that clock / thermal drift between separate runs
    (measured: up to 10 % on layers no knob touches) cancels."""
    import re
    from hover_net_b200.models.hovernet.net_desc import create_model
    nt = {"fast": 6, "original": 5}[mode]
    x = synth.make_patches(B, arch.PATCH_GEOMETRY[mode][0], seed=7)
    net = create_model(mode=mode, nr_types=nt)
    net.load_state_dict(synth.make_state_dict(mode, nt, 0))
    net.ctx.set_option("chunk", B)
    net.ctx.set_option("branch_streams", 0)
    cfgs = []
    for c in configs:
        tag, _, opts = c.partition(":")
        cfgs.append((tag, [(kv.split("=")[0], int(kv.split("=")[1])) for kv in opts.split(",") if "=" in kv]))
    keys = sorted({k for _, o in cfgs for k, _ in o})
    defaults = {"tc_prefetch": 4, "tc_xf_trunc": 1, "tc_seg_chunks": 4, "tc_block_n": 0, "xform": 1}
    net.ctx.forward(x)
    net.ctx.set_option("profile", 3)
    times = {t: {} for t, _ in cfgs}
    order = []
    for rep in range(reps):
        for tag, opts in cfgs:
            for k in keys: net.ctx.set_option(k, defaults[k])
            for k, v in opts: net.ctx.set_option(k, v)
            net.ctx.forward(x)
            seen = {}
            for l in net.ctx.debug_log().split("\n"):
                m = re.match(r"(\S+)\s+(conv_tc|conv_ref|conv0|bnrelu|head)\s.*?([\d.]+) ms", l)
                if not m: continue
                n = m.group(1); seen[n] = seen.get(n, 0) + 1
                if seen[n] > 1: n += "'" * (seen[n] - 1)
                if rep == 0 and tag == cfgs[0][0]: order.append(n)
                times[tag].setdefault(n, []).append(float(m.group(3)))
    med = {t: {n: float(np.median(v)) for n, v in d.items()} for t, d in times.items()}
    t0 = cfgs[0][0]
    print("%-46s" % ("layer (%s B=%d, median of %d)" % (mode, B, reps)) + "".join("%11s" % t for t, _ in cfgs))
    for n in order:
        vals = [med[t].get(n, float("nan")) for t, _ in cfgs]
        if any(abs(v - vals[0]) > 0.02 * vals[0] for v in vals[1:]):
            print("%-46s" % n[:46] + "".join("%11.4f" % v for v in vals))
    print("%-46s" % "TOTAL" + "".join("%11.3f" % sum(med[t].values()) for t, _ in cfgs))
    net.ctx.close()


if __name__ == "__main__" and "ab" in sys.argv[1:]:
    i = sys.argv.index("ab")
    ab(sys.argv[i + 1], int(sys.argv[i + 2]), sys.argv[i + 3:], reps=int(os.environ.get("AB_REPS", "5")))
