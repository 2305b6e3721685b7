"""Per-class breakdown of a `tools/gpu_diag.py layers <mode> <B>` log: which layer classes take the time and what bounds
each (DESIGN.md 4.1).  usage: python tools/layer_classes.py <log> [...]

Where the log carries each layer's algorithmic HBM bytes (every input read once, every output written once, weights
ignored), the table adds the class's GB and its floor: the larger of the bytes at HBM_BPS and the three fp16 products
of its FLOP (one in precision "high") at FP16_FLOPS -- H100 SXM data-sheet figures, not measured -- and floor / measured.
Logs without the bytes field print the table without those columns."""
import re
import sys

HBM_BPS = 3.35e12      # H100 SXM data sheet, HBM3
FP16_FLOPS = 989e12    # H100 SXM data sheet, dense FP16 tensor core
PRODUCTS = 3           # a_hi*w_hi + a_hi*w_lo + a_lo*w_hi per MAC


def classify(name, k, stride, cin, cout, out, bn, halo):
    if ".dense.units." in name and "conv2" in name:
        return "dense grouped kxk (128->32, g=4)"
    if k > 1:
        if cout >= 128:
            return "wide kxk (cout >= 128)"
        return "thin kxk (cout 64)"
    if name.startswith("conv_bot") or name.endswith("convf.weight"):
        return "1x1 + upsample/skip (conv_bot, convf)"
    if ".dense.units." in name:
        return "1x1 XF decoder (dense conv1)"
    if "conv1" in name and ".units.0." not in name:
        return "1x1 XF encoder (pre-activation conv1)"
    if "conv3" in name and "shortcut" not in name:
        return "1x1 + residual (conv3, d0 at full resolution)" if name.startswith("d0.") else "1x1 + residual (conv3, d1-d3)"
    if name.startswith("d0."):
        return "1x1 plain, d0 (full resolution)"
    return "1x1 plain (unit-0 conv1, conv3+shortcut)"


def main(path):
    rows = {}
    other = {}
    for l in open(path):
        m = re.match(r"(\S+)\s+conv_tc\s+k(\d)x\d s(\d) cin(\d+)\s+cout(\d+)\s+out(\d+)x\d+ box=\S+?(H?) bn=(\d+)\s+([\d.]+) ms\s+([\d.]+) GFLOP(?:\s+[\d.]+ TFLOP/s\s+([\d.]+) GB)?", l)
        if m:
            name, k, st, cin, cout, out, halo, bn, ms, gf, gb = m.groups()
            c = classify(name, int(k), int(st), int(cin), int(cout), int(out), int(bn), halo)
            r = rows.setdefault(c, [0, 0.0, 0.0, None])
            r[0] += 1; r[1] += float(ms); r[2] += float(gf)
            if gb is not None:
                r[3] = (r[3] or 0.0) + float(gb)
            continue
        m = re.match(r"(\S+)\s+(conv0|bnrelu|head)\s+([\d.]+) ms", l)
        if m:
            o = other.setdefault(m.group(2), [0, 0.0])
            o[0] += 1; o[1] += float(m.group(3))
    tot = sum(r[1] for r in rows.values())
    print("## %s  (conv_tc %.2f ms, %.0f GFLOP, %.0f TFLOP/s)" % (path, tot, sum(r[2] for r in rows.values()),
                                                              sum(r[2] for r in rows.values()) / tot))
    has_gb = all(r[3] is not None for r in rows.values())
    extra = " GB | HBM floor ms | tensor floor ms | floor / measured |" if has_gb else ""
    print("| class | launches | ms | share | GFLOP | TFLOP/s |%s\n|---|---:|---:|---:|---:|---:|%s" % (extra, "---:|" * 4 if has_gb else ""))
    for c, r in sorted(rows.items(), key=lambda x: -x[1][1]):
        line = "| %s | %d | %.3f | %.1f %% | %.0f | %.0f |" % (c, r[0], r[1], 100 * r[1] / tot, r[2], r[2] / r[1])
        if has_gb:
            hbm = r[3] * 1e9 / HBM_BPS * 1e3
            tc = PRODUCTS * r[2] * 1e9 / FP16_FLOPS * 1e3
            line += " %.2f | %.2f | %.2f | %.2f |" % (r[3], hbm, tc, max(hbm, tc) / r[1])
        print(line)
    for c, o in other.items():
        print("| (%s) | %d | %.3f | | | |%s" % (c, o[0], o[1], " | | | |" if has_gb else ""))


if __name__ == "__main__":
    for p in sys.argv[1:]:
        main(p)
