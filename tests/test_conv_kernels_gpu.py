"""The CNN kernels one operator at a time, against float64 references on the operands as stored.

The end-to-end tests compare a cropped network output; most of every intermediate tensor, its borders and its partial
tiles never reach it.  Here each kernel runs alone through tests/native/libhvn_probe.so (the engine's own objects, not
the C ABI) on shapes, views and knobs chosen to reach its edges.  Every output and residual buffer is filled with a NaN
pattern outside the view first, and must come back bit-unchanged there.

Error bound of a convolution (per output element, fp64 reference y64 of the stored operands):

    |y - y64| <= gamma * S,   S = sum_k |a_k| |w_k|   (computed alongside in fp64)

gamma follows each kernel's accumulation order (worst case, first order in the unit roundoff):
  * k_conv_tc: a segment of `tc_seg_chunks` 64-channel K-slices accumulates inside the tensor core (fp32, products of
    fp16 operands are exact); segments are summed with fp32 adds.  The tensor core aligns and truncates its additions
    (Fasi et al., "Numerical behavior of NVIDIA tensor cores", 2021), so every add is charged a full fp32 ulp, 2^-23,
    not half of one.  A segment chains P * 64 * min(seg, kiters) products (P = 3 in "highest": hi*hi + hi*lo + lo*hi,
    P = 1 in "high"), then ceil(kiters / seg) segment sums follow:
        gamma_tc = (P * 64 * min(seg, kiters) + ceil(kiters / seg)) * 2^-23  (+ 2^-21 in "highest": the lo*lo product
        the split omits is below 2^-11 * 2^-11 of |a||w|).
  * k_conv_ref: one fmaf chain over all taps and (16-padded) channels, one round-to-nearest per step:
        gamma_ref = taps * ceil16(cin) * 2^-24  (no lo*lo term: it multiplies the exact fp32 values hi + lo).
Epilogue terms scale and add to it: |BN scale| times the accumulator bound, 2^-23 of each fp32 add or fma operand,
and the fp16 storage error of a split output (2^-22 relative in "highest", 2^-11 in "high", plus half the smallest
fp16 subnormal).  The XF transform's operand (relu(x * scale + shift) formed in the kernel) differs from the fp64 one by
2^-23 (|x scale| + |shift|) plus its split: 2^-21 |y| + 2^-24 for the truncating split, one fp16 ulp (2^-10 |y| + 2^-24)
in "high"; that operand error is carried through the weights as a second convolution.

Sensitivity: with operands whose lo planes are large and of one sign (the "coherent" values below), one hi*lo product
term is about 2^-11.1 * S.  gamma_tc at 3x3, cin 64 (kiters 9, seg 4) is 771 * 2^-23 + 2^-21 = 2^-13.4, so a kernel
that drops that term exceeds its bound about 4.7 times over (measured by removing the a_lo * w_hi product).
"""
import ctypes
import math
import os
import re
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
U = 2.0 ** -24
NAN16 = 0x7E5A                      # fp16 NaN canary
NAN32 = 0x7FC05A5A                  # fp32 NaN canary
DEFAULT_KNOBS = (0, 4, 4, 1)        # tc_block_n, tc_seg_chunks, tc_prefetch, tc_xf_trunc as the engine starts
EPI = {"PLAIN": 0, "RES": 1, "UP2": 2}
DISPATCHED = set()                  # (BLOCK_N, epilogue, XF, ONE) over the module
RATIOS = []


# ------------------------------------------------------------------------------------------------ probe and buffers
@pytest.fixture(scope="module")
def probe():
    if not torch.cuda.is_available():
        pytest.fail("needs a CUDA device")
    sys.path.insert(0, os.path.join(HERE, "native"))
    try:
        import build_probe
    finally:
        sys.path.pop(0)
    from hover_net_b200 import build
    build.build()
    L = ctypes.CDLL(build_probe.build())
    i64p, i32p = ctypes.POINTER(ctypes.c_longlong), ctypes.POINTER(ctypes.c_int)
    L.probe_conv.argtypes = [i64p, ctypes.c_int, i32p]
    L.probe_conv0.argtypes = [ctypes.c_longlong] + [ctypes.c_int] * 5 + [ctypes.c_longlong] * 6 + [i64p, ctypes.c_longlong]
    L.probe_bnrelu.argtypes = [i64p, ctypes.c_int, ctypes.c_longlong, ctypes.c_longlong, i64p, ctypes.c_longlong]
    L.probe_up2_add.argtypes = [i64p, ctypes.c_int, i64p, i64p, ctypes.c_longlong]
    L.probe_head.argtypes = [ctypes.c_int, i64p, i64p, i64p, i32p, i32p] + [ctypes.c_int] * 4 + [ctypes.c_longlong]
    L.probe_set_knobs.argtypes = [ctypes.c_int] * 4
    L.probe_set_knobs(*DEFAULT_KNOBS)
    yield L
    L.probe_set_knobs(*DEFAULT_KNOBS)


def _i64(v):
    return (ctypes.c_longlong * len(v))(*[int(x) for x in v])


class Split:
    """Split (hi, lo) NHWC buffer [B, Hb, Wb, Cb] filled with the NaN canary, with a view at (y0, x0, c0)."""

    def __init__(self, B, Hb, Wb, Cb, one, view=None):
        self.hi = torch.full((B, Hb, Wb, Cb), NAN16, dtype=torch.int16, device="cuda").view(torch.float16)
        self.lo = None if one else torch.full_like(self.hi.view(torch.int16), NAN16).view(torch.float16)
        self.view_at(*(view or (0, 0, 0, Hb, Wb, Cb)))

    def view_at(self, y0, x0, c0, h, w, c):
        self.v = (y0, x0, c0, h, w, c)
        return self

    def sl(self, t):
        y0, x0, c0, h, w, c = self.v
        return t[:, y0:y0 + h, x0:x0 + w, c0:c0 + c]

    def desc(self):
        hv = self.sl(self.hi)
        s = self.hi.stride()
        return [hv.data_ptr(), 0 if self.lo is None else self.sl(self.lo).data_ptr(), s[0], s[1], s[2]] + list(self.v[3:])

    def fill(self, hi, lo=None):
        self.sl(self.hi).copy_(hi)
        if self.lo is not None:
            self.sl(self.lo).copy_(lo)

    def value(self):
        v = self.sl(self.hi).double()
        return v if self.lo is None else v + self.sl(self.lo).double()

    def canaries_intact(self):
        for t in (self.hi, self.lo):
            if t is None:
                continue
            m = torch.ones(t.shape, dtype=torch.bool, device="cuda")
            self.sl(m).fill_(False)
            if not bool((t.view(torch.int16)[m] == NAN16).all()):
                return False
        return True


class Raw:
    def __init__(self, B, Hb, Wb, Cb, view=None):
        self.p = torch.full((B, Hb, Wb, Cb), NAN32, dtype=torch.int32, device="cuda").view(torch.float32)
        self.v = view or (0, 0, 0, Hb, Wb, Cb)

    def sl(self, t):
        y0, x0, c0, h, w, c = self.v
        return t[:, y0:y0 + h, x0:x0 + w, c0:c0 + c]

    def desc(self):
        s = self.p.stride()
        return [self.sl(self.p).data_ptr(), 0, s[0], s[1], s[2]] + list(self.v[3:])

    def canaries_intact(self):
        m = torch.ones(self.p.shape, dtype=torch.bool, device="cuda")
        self.sl(m).fill_(False)
        return bool((self.p.view(torch.int32)[m] == NAN32).all())


# ------------------------------------------------------------------------------------------------ host restatements
def split_host(x32):
    """split_f32 on the host: hi = fp16_rn(x), lo = fp16_rn(x - hi) (x - hi is exact in fp32)."""
    hi = x32.half()
    return hi, (x32 - hi.float()).half()


def tf_same_lo(size, k, stride):
    """TF-"same" padding above / left of the image (reference net_utils.py:51-63, restated in cnn.cu)."""
    pad = max(k - stride, 0) if size % stride == 0 else max(k - size % stride, 0)
    return pad // 2


def weight_planes(w32, one, device="cuda"):
    """Model::make_conv: OIHW fp32 -> [tap][cout][cin_pad] fp16 planes of w * 2^e[cout], e putting the channel's max |w|
    in [2^13, 2^14); returns (hi, lo, oscale, stored OIHW fp64)."""
    O, I, kh, kw = w32.shape
    mx = w32.abs().amax(dim=(1, 2, 3)).double()
    e = torch.where(mx > 0, 14 - torch.frexp(mx).exponent, torch.zeros_like(mx, dtype=torch.int32))
    v = w32 * torch.pow(2.0, e.float()).view(O, 1, 1, 1)
    hi, lo = split_host(v)
    cin_pad = (I + 63) // 64 * 64
    stored = hi.double() + (0 if one else lo.double())
    stored = stored * torch.pow(2.0, -e.double()).view(O, 1, 1, 1)

    def planes(t):
        p = torch.zeros(kh * kw, O, cin_pad, dtype=torch.float16)
        p[:, :, :I] = t.permute(2, 3, 0, 1).reshape(kh * kw, O, I)
        return p.to(device)

    return planes(hi), None if one else planes(lo), torch.pow(2.0, -e.float()).to(device), stored.to(device)


def conv64(a, w, stride, pad, ho, wo):
    """fp64 NHWC convolution over a zero-padded view: a [B,h,w,c], w OIHW -> [B,ho,wo,O]."""
    B, h, wd, c = a.shape
    kh, kw = w.shape[2:]
    pb = max(0, (ho - 1) * stride + kh - pad - h)
    pr = max(0, (wo - 1) * stride + kw - pad - wd)
    x = F.pad(a.permute(0, 3, 1, 2), (pad, pr, pad, pb))
    return F.conv2d(x, w.double(), stride=stride)[:, :, :ho, :wo].permute(0, 2, 3, 1)


def values(shape, kind, gen):
    """Operand values: 'normal', 'wide' (|x| from 2^-20 to 2^10 with exact zeros), 'coherent' (positive, lo planes
    about 2^-11 of hi and of one sign), 'pos' (uniform [0, 1))."""
    if kind == "normal":
        return torch.randn(shape, generator=gen)
    if kind == "pos":
        return torch.rand(shape, generator=gen)
    if kind == "wide":
        mag = torch.pow(2.0, torch.empty(shape).uniform_(-20, 10, generator=gen))
        x = mag * torch.sign(torch.randn(shape, generator=gen))
        return torch.where(torch.rand(shape, generator=gen) < 0.1, torch.zeros_like(x), x)
    if kind == "coherent":  # hi in [1, 1.25) (fp16 ulp 2^-10), x = hi + 0.499 ulp -> lo = 2^-11 of |x|, all positive
        hi = 1.0 + torch.randint(0, 256, shape, generator=gen).float() * 2.0 ** -10
        return hi + 0.499 * 2.0 ** -10
    raise ValueError(kind)


# ------------------------------------------------------------------------------------------------ convolution runner
def gamma_tc(one, taps, cin_pad, seg):
    kiters = taps * cin_pad // 64
    n = (1 if one else 3) * 64 * min(seg, kiters) + math.ceil(kiters / seg)
    return n * 2.0 ** -23 + (0.0 if one else 2.0 ** -21)


def gamma_ref(taps, cin):
    return taps * ((cin + 15) // 16 * 16) * U


def run_conv(L, *, path, prec, B, h, w, cin, cout, k=1, stride=1, pad=0, ho=None, wo=None, a_view=None,
             out="raw", out_c=None, bn=False, relu=False, res=None, up2=False, skip_crop=0, a2=None, xf=None,
             vals="normal", wvals="normal", wscale=False, groups=1, seed=0, knobs=DEFAULT_KNOBS, expect=None):
    """One convolution through k_conv_tc (path 'tc') or k_conv_ref (path 'ref') against its fp64 reference.

    a_view: (Hb, Wb, Cb, y0, x0, c0) of a wider input buffer.  out: 'raw', 'split' or 'both'; out_c = (Cb, c0) writes a
    channel window.  res: None, 'sep' or 'alias' (res is out_raw).  a2 = dict(c, stride, box): fused shortcut source.
    xf = dict(trunc, tail_nan): the input is a raw fp32 tensor transformed by relu(x * scale + shift) in the kernel."""
    one = prec == "high"
    gen = torch.Generator().manual_seed(seed)
    ho = ho if ho is not None else (h + 2 * pad - k) // stride + 1
    wo = wo if wo is not None else (w + 2 * pad - k) // stride + 1
    Hb, Wb, Cb, y0, x0, c0 = a_view or (h, w, cin, 0, 0, 0)
    d = [0] * 80
    d[70], d[72], d[73], d[74], d[75], d[76], d[77] = 1, stride, pad, pad, B, ho, wo
    keep = []
    a_err = None
    # ---- input
    if xf is None:
        A = Split(B, Hb, Wb, Cb, one).view_at(y0, x0, c0, h, w, cin)
        x32 = values((B, h, w, cin), vals, gen)
        if one:
            A.fill(x32.half().cuda())
        else:
            A.fill(*[t.cuda() for t in split_host(x32)])
        a64 = A.value()
        d[0:8] = A.desc()
    else:
        R = Raw(B, Hb, Wb, Cb, (y0, x0, c0, h, w, cin))
        x32 = values((B, h, w, cin), vals, gen)
        R.sl(R.p).copy_(x32.cuda())
        sc = (torch.rand(cin, generator=gen) + 0.5)
        sh = torch.randn(cin, generator=gen) * 0.7          # about half the inputs negative before the ReLU
        tail = 64
        scb = torch.full((cin + tail,), float("nan") if xf.get("tail_nan", True) else 0.0)
        shb = scb.clone()
        scb[:cin], shb[:cin] = sc, sh
        scb, shb = scb.cuda(), shb.cuda()
        keep += [R, scb, shb]
        xs = x32.double().cuda() * sc.double().cuda()
        a64 = torch.clamp(xs + sh.double().cuda(), min=0)
        if one:
            a_err = 2.0 ** -23 * (xs.abs() + sh.double().cuda().abs()) + 2.0 ** -10 * a64 + 2.0 ** -24
        else:
            a_err = 2.0 ** -23 * (xs.abs() + sh.double().cuda().abs()) + 2.0 ** -21 * a64 + 2.0 ** -24
        A = Split(B, h, w, cin, one)                         # the referee's materialised operand (and the range flag)
        d[0:8] = A.desc()
        d[8:16] = R.desc()
        d[65], d[66] = scb.data_ptr(), shb.data_ptr()
    keep.append(A)
    # ---- weights
    w32 = values((cout, cin // groups, k, k), wvals, gen) * 0.1
    if groups > 1:
        full = torch.zeros(cout, cin, k, k)
        og, ig = cout // groups, cin // groups
        for g in range(groups):
            full[g * og:(g + 1) * og, g * ig:(g + 1) * ig] = w32[g * og:(g + 1) * og]
        w32 = full
    if wscale:  # per-output-channel scales 2^-8 .. 2^8
        w32 = w32 * torch.pow(2.0, torch.randint(-8, 9, (cout, 1, 1, 1), generator=gen).float())
    cin_tot = cin
    if a2 is not None:
        s2 = a2["stride"]
        h2, w2 = a2.get("h", ho * s2), a2.get("w", wo * s2)
        A2b = a2.get("buf")
        if A2b:
            A2 = Split(B, A2b[0], A2b[1], A2b[2], one).view_at(A2b[3], A2b[4], A2b[5], h2, w2, a2["c"])
        else:
            A2 = Split(B, h2, w2, a2["c"], one)
        x2 = values((B, h2, w2, a2["c"]), vals, gen)
        if one:
            A2.fill(x2.half().cuda())
        else:
            A2.fill(*[t.cuda() for t in split_host(x2)])
        keep.append(A2)
        d[16:24] = A2.desc()
        d[70], d[71] = s2, cin
        w2_32 = values((cout, a2["c"], 1, 1), wvals, gen) * 0.1
        w32 = torch.cat([w32, w2_32], 1)
        cin_tot = cin + a2["c"]
    whi, wlo, osc, wst = weight_planes(w32, one)
    keep += [whi, wlo, osc]
    d[56], d[57], d[58] = whi.data_ptr(), 0 if wlo is None else wlo.data_ptr(), osc.data_ptr()
    d[59], d[60], d[61], d[62], d[63], d[64] = k * k, cout, cin_tot, whi.shape[2], k, k
    # ---- fp64 reference of the accumulator and its bound
    y64 = conv64(a64, wst[:, :cin], stride, pad, ho, wo)
    S = conv64(a64.abs(), wst[:, :cin].abs(), stride, pad, ho, wo)
    extra = torch.zeros_like(S)
    if a_err is not None:
        extra = conv64(a_err, wst[:, :cin].abs(), stride, pad, ho, wo)
    if a2 is not None:
        a2v = A2.value()[:, ::s2, ::s2][:, :ho, :wo]
        y64 = y64 + conv64(a2v, wst[:, cin:], 1, 0, ho, wo)
        S = S + conv64(a2v.abs(), wst[:, cin:].abs(), 1, 0, ho, wo)
    seg = knobs[1]
    if path == "tc":
        g = gamma_tc(one, k * k, whi.shape[2], seg)
    else:
        g = gamma_ref(k * k, cin) + (gamma_ref(1, a2["c"]) if a2 else 0.0)
    acc_bound = g * S + extra
    # ---- epilogue operands
    outs = []
    raw64, raw_bound = y64, acc_bound
    if res is not None:
        r32 = values((B, ho, wo, cout), "normal", gen)
        if res == "alias":
            OR = Raw(B, ho, wo, cout)
            OR.sl(OR.p).copy_(r32.cuda())
            RS = OR
        else:
            RS = Raw(B, ho + 2, wo + 1, cout + 32, (1, 1, 16, ho, wo, cout))
            RS.sl(RS.p).copy_(r32.cuda())
            keep.append(RS)
        d[24:32] = RS.desc()
        raw64 = y64 + r32.double().cuda()
        raw_bound = acc_bound + 2.0 ** -23 * raw64.abs()
    if out in ("raw", "both"):
        if res != "alias":
            OC, oc0 = out_c or (cout, 0)
            OR = Raw(B, ho + 3, wo + 2, OC, (2, 1, oc0, ho, wo, cout))
        d[32:40] = OR.desc()
        outs.append(("raw", OR, raw64, raw_bound))
    sc_b = sh_b = None
    if up2:
        SK = Split(B, 2 * ho + 2 * skip_crop, 2 * wo + 2 * skip_crop, cout, one).view_at(skip_crop, skip_crop, 0, 2 * ho, 2 * wo, cout)
        s32 = values((B, 2 * ho, 2 * wo, cout), "normal", gen)
        if one:
            SK.fill(s32.half().cuda())
        else:
            SK.fill(*[t.cuda() for t in split_host(s32)])
        keep.append(SK)
        d[48:56] = SK.desc()
        d[79] = 1
        OS = Split(B, 2 * ho + 1, 2 * wo + 3, cout + 16, one).view_at(1, 2, 8, 2 * ho, 2 * wo, cout)
        d[40:48] = OS.desc()
        up = raw64.repeat_interleave(2, 1).repeat_interleave(2, 2)
        t64 = up + SK.value()
        tb = raw_bound.repeat_interleave(2, 1).repeat_interleave(2, 2) + 2.0 ** -23 * t64.abs()
        outs.append(("split", OS, t64, tb))
    elif out in ("split", "both"):
        OC, oc0 = out_c or (cout, 0)
        OS = Split(B, ho + 1, wo + 2, OC, one).view_at(1, 1, oc0, ho, wo, cout)
        d[40:48] = OS.desc()
        t64, tb = raw64, raw_bound
        if bn:
            sc_b = (torch.rand(cout, generator=gen) + 0.5).cuda()
            sh_b = (torch.randn(cout, generator=gen) * 0.1).cuda()
            keep += [sc_b, sh_b]
            d[67], d[68] = sc_b.data_ptr(), sh_b.data_ptr()
            ts = raw64 * sc_b.double()
            t64 = ts + sh_b.double()
            tb = raw_bound * sc_b.double() + 2.0 ** -23 * (ts.abs() + sh_b.double().abs())
        if relu:
            d[78] = 1
            t64 = t64.clamp(min=0)
        outs.append(("split", OS, t64, tb))
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    d[69] = flag.data_ptr()
    info = (ctypes.c_int * 10)()
    L.probe_set_knobs(*knobs)
    try:
        torch.cuda.synchronize()
        rc = L.probe_conv(_i64(d), 0 if path == "tc" else 1, info)
    finally:
        L.probe_set_knobs(*DEFAULT_KNOBS)
    assert rc == 0, "probe_conv returned %d (1: tc_plan declined the layer)" % rc
    info = list(info)
    if path == "tc":
        assert info[0] == 1 and info[5] == int(one)
        disp = (info[9], info[6], info[7], info[8])
        assert disp[0] == info[1] and disp[3] == int(one) and disp[2] == int(xf is not None)
        want_epi = "UP2" if up2 else ("RES" if res else "PLAIN")
        assert disp[1] == EPI[want_epi], (disp, want_epi)
        DISPATCHED.add(disp)
        if expect:
            for key, val in expect.items():
                got = {"block_n": info[1], "flat": info[2], "bw": info[3], "bh": info[4]}[key]
                assert got == val, "%s = %d, expected %d" % (key, got, val)
    assert int(flag.item()) == 0, "range flag raised on in-range data"
    worst, worst_b = None, 0.0
    for kind, buf, ref, bound in outs:
        got = buf.sl(buf.p).double() if kind == "raw" else buf.value()
        if kind == "split":  # storage of a split (or single-plane) output
            bound = bound + (2.0 ** -11 if one else 2.0 ** -22) * ref.abs() + 2.0 ** -25
        assert torch.isfinite(got).all(), "%s output has non-finite values" % kind
        err = (got - ref).abs()
        over = err > bound
        assert not bool(over.any()), "%s: %d elements over the bound, worst err/bound %.3g" % (
            kind, int(over.sum()), float((err / bound.clamp(min=1e-300)).max()))
        worst_b = max(worst_b, float((err / bound.clamp(min=1e-300)).max()))
        if kind == "raw":  # the accumulator's own error, in units of S * 2^-24 (elements with S > 0)
            r = err[S > 0] / S[S > 0] / U
            worst = max(worst or 0.0, float(r.max()) if r.numel() else 0.0)
        assert buf.canaries_intact(), "%s buffer written outside its view" % kind
    for b in keep:
        if isinstance(b, (Split, Raw)):
            assert b.canaries_intact(), "an input buffer changed outside its view"
    if worst is not None:
        RATIOS.append((worst, g / U, path, prec, xf is not None))
    print("  %-4s %-7s raw err/(S*2^-24) = %9s   gamma/2^-24 = %8.1f   worst err/bound = %.3f   plan bn=%d flat=%d box=%dx%d" % (
        path, prec, "-" if worst is None else "%.2f" % worst, g / U, worst_b, info[1], info[2], info[3], info[4]))
    return info, outs


PRECS = ["highest", "high"]
PATHS = ["tc", "ref"]


def both(L, **kw):
    for prec in PRECS:
        for path in PATHS:
            run_conv(L, path=path, prec=prec, **kw)


# ------------------------------------------------------------------------------------------------ b. flat path
@pytest.mark.parametrize("case", [
    dict(B=1, h=5, w=7, cin=64, cout=32, out="both", bn=True, relu=True, expect=dict(flat=1, block_n=32)),  # m_total 35
    dict(B=3, h=33, w=33, cin=128, cout=64, expect=dict(flat=1, block_n=64)),        # tiles span two images
    dict(B=2, h=96, w=96, cin=64, cout=256, out="both", bn=True, expect=dict(flat=1, block_n=128)),  # 288 tiles > SMs
    dict(B=1, h=12, w=12, cin=2048, cout=128, up2=True, skip_crop=3, vals="wide", expect=dict(flat=1)),  # K of conv_bot
], ids=["m35", "two_images", "many_tiles_kiters1", "cin2048_up2"])
def test_flat_path(probe, case):
    both(probe, **case)


def test_prefetch_is_only_a_hint(probe):
    """tc_prefetch 0, 4 and 100 (past kiters = 8): bit-identical outputs."""
    res = []
    for pf in (0, 4, 100):
        _, outs = run_conv(probe, path="tc", prec="highest", B=2, h=40, w=40, cin=512, cout=128, out="both", bn=True,
                           knobs=(0, 4, pf, 1), expect=dict(flat=1))
        res.append([b.p.clone() if k == "raw" else b.hi.clone() for k, b, _, _ in outs])
    for r in res[1:]:
        assert all(torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x.view(torch.int16),
                               y.view(torch.int32) if y.dtype == torch.float32 else y.view(torch.int16))
                   for x, y in zip(res[0], r))


# ------------------------------------------------------------------------------------------------ c. 4-D box path
@pytest.mark.parametrize("case", [
    dict(B=2, h=17, w=19, cin=64, cout=64, k=3, pad=1, res="sep", expect=dict(flat=0, block_n=64)),
    dict(B=1, h=13, w=11, cin=64, cout=32, k=5, pad=2, out="split", bn=True, relu=True, expect=dict(flat=0)),
    dict(B=2, h=14, w=15, cin=128, cout=128, k=3, pad=0, expect=dict(flat=0)),                     # valid 3x3
    dict(B=1, h=20, w=18, cin=64, cout=64, k=5, pad=0, vals="coherent", wvals="pos", expect=dict(flat=0)),  # valid 5x5
    dict(B=2, h=16, w=16, cin=64, cout=128, k=3, stride=2, pad=tf_same_lo(16, 3, 2), ho=8, wo=8, expect=dict(flat=0)),
    dict(B=2, h=15, w=15, cin=64, cout=128, k=3, stride=2, pad=tf_same_lo(15, 3, 2), ho=8, wo=8, expect=dict(flat=0)),
    dict(B=2, h=16, w=15, cin=128, cout=256, k=1, stride=2, ho=8, wo=8, expect=dict(flat=0)),     # unfused shortcut
    dict(B=1, h=7, w=13, cin=64, cout=64, k=3, pad=1, expect=dict(flat=0)),
    dict(B=2, h=37, w=37, cin=64, cout=32, k=3, pad=1, res="sep", expect=dict(flat=0)),
    dict(B=2, h=1, w=200, cin=64, cout=64, k=3, pad=1, expect=dict(flat=0)),
    dict(B=2, h=200, w=1, cin=64, cout=128, k=3, pad=1, res="sep", expect=dict(flat=0)),
    dict(B=1, h=3, w=150, cin=64, cout=128, k=3, pad=1, up2=True, expect=dict(flat=0)),          # wo > 128
], ids=["3x3p1_res", "5x5p2", "valid3", "valid5_coherent", "s2_even", "s2_odd_same", "1x1s2", "7x13", "37x37_res",
        "1x200", "200x1_res", "wo150_up2"])
def test_box_path(probe, case):
    both(probe, **case)


# ------------------------------------------------------------------------------------------------ d. views
@pytest.mark.parametrize("case", [
    # dense concat: channel window 288 of 512 at a spatial offset; the last K-slice is partly past the view
    dict(B=2, h=14, w=14, cin=288, cout=128, a_view=(20, 20, 512, 2, 3, 0), out="split", bn=True, relu=True,
         expect=dict(flat=0, block_n=128)),
    dict(B=2, h=9, w=10, cin=32, cout=64, k=3, pad=1, expect=dict(flat=0)),
    dict(B=2, h=12, w=12, cin=96, cout=32, expect=dict(flat=1, block_n=32)),
    # a dense unit's grouped conv2 (block-diagonal 128 -> 32, valid 5x5) into a 32-channel window of the concat buffer
    dict(B=2, h=15, w=15, cin=128, cout=32, k=5, groups=4, out_c=(352, 288), expect=dict(flat=0, block_n=32)),
    dict(B=2, h=16, w=16, cin=128, cout=256, res="alias", out="both", bn=True, relu=True, expect=dict(flat=1)),
    dict(B=2, h=10, w=11, cin=64, cout=32, k=3, pad=1, up2=True, skip_crop=4, vals="wide", expect=dict(block_n=32)),
    dict(B=1, h=24, w=24, cin=256, cout=64, up2=True, skip_crop=2, a_view=(24, 30, 256, 0, 3, 0), expect=dict(flat=0)),
], ids=["concat288of512", "cin32", "cin96", "window32", "res_alias", "up2_crop", "up2_box"])
def test_views(probe, case):
    both(probe, **case)


# ------------------------------------------------------------------------------------------------ e. fused shortcut
@pytest.mark.parametrize("case", [
    dict(B=2, h=16, w=16, cin=64, cout=256, a2=dict(c=128, stride=1), res=None, out="both", bn=True, expect=dict(flat=1)),
    dict(B=2, h=16, w=16, cin=64, cout=256, a_view=(18, 18, 64, 1, 1, 0), a2=dict(c=128, stride=1),
         expect=dict(flat=0)),
    dict(B=2, h=8, w=8, cin=128, cout=512, a2=dict(c=256, stride=2), out="both", bn=True, expect=dict(flat=0)),
    dict(B=1, h=8, w=8, cin=128, cout=512, a2=dict(c=256, stride=2, h=15, w=15), expect=dict(flat=0)),  # odd source
], ids=["flat_s1", "box_s1", "box_s2", "box_s2_odd"])
def test_fused_shortcut(probe, case):
    both(probe, **case)


# ------------------------------------------------------------------------------------------------ f. XF
@pytest.mark.parametrize("trunc", [1, 0])
@pytest.mark.parametrize("case", [
    dict(B=2, h=20, w=20, cin=256, cout=128, out="split", bn=True, relu=True, expect=dict(flat=1, block_n=128)),
    dict(B=2, h=13, w=13, cin=288, cout=64, a_view=(17, 17, 512, 2, 2, 0), out="split", bn=True, relu=True,
         expect=dict(flat=0, block_n=64)),
    dict(B=1, h=9, w=9, cin=160, cout=128, up2=True, skip_crop=3, expect=dict(flat=1, block_n=128)),
    dict(B=2, h=7, w=7, cin=224, cout=64, a_view=(11, 11, 256, 2, 2, 0), up2=True, expect=dict(flat=0, block_n=64)),
], ids=["flat_bn128", "box_bn64", "flat_up2", "box_up2"])
def test_xf_transform(probe, case, trunc):
    for prec in PRECS:
        for path in PATHS:
            run_conv(probe, path=path, prec=prec, xf=dict(trunc=trunc, tail_nan=True), knobs=(0, 4, 4, trunc),
                     vals="normal", **case)


# ------------------------------------------------------------------------------------------------ g. knobs
@pytest.mark.parametrize("bn", [32, 64])
def test_forced_block_n(probe, bn):
    for prec in PRECS:
        run_conv(probe, path="tc", prec=prec, B=2, h=12, w=12, cin=128, cout=256, k=3, pad=1, res="sep", knobs=(bn, 4, 4, 1),
                 expect=dict(block_n=bn))
        run_conv(probe, path="tc", prec=prec, B=1, h=10, w=10, cin=64, cout=256, up2=True, knobs=(bn, 4, 4, 1),
                 expect=dict(block_n=bn))


@pytest.mark.parametrize("seg", [1, 3, 1000])
def test_seg_chunks(probe, seg):
    for prec in PRECS:
        run_conv(probe, path="tc", prec=prec, B=1, h=10, w=10, cin=512, cout=128, k=3, pad=1, vals="wide", wscale=True,
                 knobs=(0, seg, 4, 1))


# ------------------------------------------------------------------------------------------------ h. operand values
@pytest.mark.parametrize("vals,wvals,wscale,out", [("wide", "normal", False, "both"), ("wide", "normal", True, "raw"),
                                                   ("coherent", "pos", False, "both"), ("pos", "wide", True, "raw")])
def test_operand_values(probe, vals, wvals, wscale, out):
    """Per-channel weight scales 2^-8 .. 2^8 take sums past fp16's range: those cases check the raw fp32 output."""
    both(probe, B=2, h=11, w=12, cin=64, cout=128, k=3, pad=1, vals=vals, wvals=wvals, wscale=wscale, out=out,
         bn=True)


# ------------------------------------------------------------------------------------------------ i. stems
def _stem_weights(w32, one):
    """finalize's two stem layouts: [64][192] planes (k = ky*24 + kx*3 + ch) with the channel exponent, and fp32
    [ky][kx][ch][64] (fp16-rounded under the exponent in "high"); plus the stored OIHW fp64 weights of each."""
    mx = w32.abs().amax(dim=(1, 2, 3)).double()
    e = torch.where(mx > 0, 14 - torch.frexp(mx).exponent, torch.zeros_like(mx, dtype=torch.int32))
    scale = torch.pow(2.0, e.float()).view(64, 1, 1, 1)
    hi, lo = split_host(w32 * scale)
    tc_st = (hi.double() + (0 if one else lo.double())) / scale.double()
    ph = torch.zeros(64, 192, dtype=torch.float16)
    pl = torch.zeros(64, 192, dtype=torch.float16)
    for ky in range(7):
        for kx in range(7):
            for ch in range(3):
                ph[:, ky * 24 + kx * 3 + ch] = hi[:, ch, ky, kx]
                pl[:, ky * 24 + kx * 3 + ch] = lo[:, ch, ky, kx]
    core = (hi.float() / scale) if one else w32
    return ph.cuda(), None if one else pl.cuda(), torch.pow(2.0, -e.float()).cuda(), tc_st.cuda(), \
        core.permute(2, 3, 1, 0).contiguous().cuda(), core.double().cuda()


@pytest.mark.parametrize("mode,B,H,W", [("fast", 2, 128, 128), ("original", 1, 134, 134), ("fast", 1, 270, 270),
                                        ("fast", 2, 140, 128), ("original", 3, 166, 166)],
                         ids=["fast128", "orig134", "fast270_strip831", "HneW", "many_tiles"])
def test_stems(probe, mode, B, H, W):
    pad = 3 if mode == "fast" else 0
    ho, wo = H + 2 * pad - 6, W + 2 * pad - 6
    gen = torch.Generator().manual_seed(H * 7 + B)
    img = torch.randint(0, 256, (B, H, W, 3), generator=gen, dtype=torch.uint8)
    img[0, :9] = 255
    img[-1, -5:, :, :] = 0
    img[:, :, -7:] = 0
    imgd = img.cuda()
    w32 = torch.randn(64, 3, 7, 7, generator=gen) * 0.1
    sc = (torch.rand(64, generator=gen) + 0.5).cuda()
    sh = (torch.randn(64, generator=gen) * 0.1).cuda()
    for prec in PRECS:
        one = prec == "high"
        ph, pl, osc, tc_st, core_w, core_st = _stem_weights(w32, one)
        xf32 = (img.float() / 255.0)
        for path in (0, 1):
            if path == 0:
                hi, lo = split_host(xf32)
                a64 = (hi.double() + (0 if one else lo.double())).cuda()
                wst, n, u = tc_st, (1 if one else 3) * 192, 2.0 ** -23
            else:
                a64 = (xf32.half().double() if one else xf32.double()).cuda()
                wst, n, u = core_st, 147, U
            y = conv64(a64, wst, 1, pad, ho, wo)
            S = conv64(a64.abs(), wst.abs(), 1, pad, ho, wo)
            ts = y * sc.double()
            t64 = (ts + sh.double()).clamp(min=0)
            bound = (n * u + (0 if one or path else 2.0 ** -21)) * S * sc.double() + 2.0 ** -22 * (ts.abs() + sh.double().abs())
            bound = bound + (2.0 ** -11 if one else 2.0 ** -22) * t64 + 2.0 ** -25
            O = Split(B, ho + 2, wo + 1, 64 + 8, one).view_at(1, 1, 8, ho, wo, 64)
            flag = torch.zeros(1, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            rc = probe.probe_conv0(imgd.data_ptr(), B, H, W, pad, path, ph.data_ptr(), 0 if pl is None else pl.data_ptr(),
                                   osc.data_ptr(), core_w.data_ptr(), sc.data_ptr(), sh.data_ptr(), _i64(O.desc()),
                                   flag.data_ptr())
            assert rc == 0, "probe_conv0 returned %d (1: the tensor-core stem declined the shape)" % rc
            assert int(flag.item()) == 0
            err = (O.value() - t64).abs()
            assert bool((err <= bound).all()), "%s path %d: worst err/bound %.3g" % (prec, path, float((err / bound).max()))
            assert O.canaries_intact()
            print("  stem path %d %-7s worst err/bound = %.3f" % (path, prec, float((err / bound).max())))


# ------------------------------------------------------------------------------------------------ j. elementwise, heads
def test_bnrelu_and_up2_add(probe):
    gen = torch.Generator().manual_seed(3)
    B, h, w, c = 2, 9, 11, 96
    for prec in PRECS:
        one = prec == "high"
        R = Raw(B, h + 2, w + 3, 160, (1, 2, 32, h, w, c))
        x = values((B, h, w, c), "wide", gen).cuda()
        R.sl(R.p).copy_(x)
        sc, sh = (torch.randn(c, generator=gen)).cuda(), (torch.randn(c, generator=gen) * 0.01).cuda()
        O = Split(B, h + 1, w + 1, 128, one).view_at(1, 0, 16, h, w, c)
        flag = torch.zeros(1, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        assert probe.probe_bnrelu(_i64(R.desc()), B, sc.data_ptr(), sh.data_ptr(), _i64(O.desc()), flag.data_ptr()) == 0
        xs = x.double() * sc.double()
        t = (xs + sh.double()).clamp(min=0)
        bound = 2.0 ** -23 * (xs.abs() + sh.double().abs()) + (2.0 ** -11 if one else 2.0 ** -22) * t + 2.0 ** -25
        assert bool(((O.value() - t).abs() <= bound).all()) and O.canaries_intact() and R.canaries_intact()
        assert int(flag.item()) == 0
        # 2x nearest upsample + skip add, channel windows on all three tensors
        R2 = Raw(B, h + 1, w, 72, (1, 0, 8, h, w, 64))
        x2 = values((B, h, w, 64), "normal", gen).cuda()
        R2.sl(R2.p).copy_(x2)
        SK = Split(B, 2 * h + 4, 2 * w + 4, 80, one).view_at(2, 2, 16, 2 * h, 2 * w, 64)
        s32 = values((B, 2 * h, 2 * w, 64), "wide", gen)
        if one:
            SK.fill(s32.half().cuda())
        else:
            SK.fill(*[t_.cuda() for t_ in split_host(s32)])
        O2 = Split(B, 2 * h, 2 * w + 2, 64, one).view_at(0, 1, 0, 2 * h, 2 * w, 64)
        torch.cuda.synchronize()
        assert probe.probe_up2_add(_i64(R2.desc()), B, _i64(SK.desc()), _i64(O2.desc()), flag.data_ptr()) == 0
        t = x2.double().repeat_interleave(2, 1).repeat_interleave(2, 2) + SK.value()
        bound = 2.0 ** -24 * t.abs() + (2.0 ** -11 if one else 2.0 ** -22) * t.abs() + 2.0 ** -25
        assert bool(((O2.value() - t).abs() <= bound).all()) and O2.canaries_intact() and SK.canaries_intact()
        assert int(flag.item()) == 0


@pytest.mark.parametrize("nt", [1, 2, 16])
def test_heads(probe, nt):
    """k_head: TP argmax (first maximal index), NP softmax probability, HV regression, per branch, on split features."""
    gen = torch.Generator().manual_seed(nt)
    B, h, w = 2, 13, 17
    feats, ws, bs, kinds, chans = [], [], [], [], []
    for kind, och in ((0, nt), (1, 2), (2, 2)):
        f32 = values((B, h, w, 64), "pos", gen)
        f32[0, :4] = 0                                      # exact ties below: zero features
        F_ = Split(B, h, w + 1, 96, False).view_at(0, 1, 16, h, w, 64)
        F_.fill(*[t.cuda() for t in split_host(f32)])
        wt = (torch.randn(och, 64, generator=gen) * 0.2).cuda()
        bias = torch.randn(och, generator=gen).cuda()
        if kind == 0 and nt > 1:
            bias[: nt] = bias[: nt].max()                   # equal biases: every zero-feature pixel is an exact tie
        feats.append(F_); ws.append(wt); bs.append(bias); kinds.append(kind); chans.append(och)
    C = 4
    out = torch.full((B, h, w, C), float("nan"), device="cuda")
    torch.cuda.synchronize()
    rc = probe.probe_head(3, _i64(sum((f.desc() for f in feats), [])), _i64([t.data_ptr() for t in ws]),
                          _i64([t.data_ptr() for t in bs]), (ctypes.c_int * 3)(*chans), (ctypes.c_int * 3)(*kinds),
                          B, h, w, C, out.data_ptr())
    assert rc == 0
    logits = [torch.einsum("bhwc,oc->bhwo", f.value(), wt.double()) + b.double() for f, wt, b in zip(feats, ws, bs)]
    tp = logits[0]
    top2 = tp.topk(min(2, nt), -1).values
    clear = (top2[..., 0] - top2[..., -1] > 1e-4) if nt > 1 else torch.ones_like(top2[..., 0], dtype=torch.bool)
    ties = (feats[0].value() == 0).all(-1)
    want = tp.argmax(-1).float()
    got = out[..., 0].double()
    assert bool((got[clear | ties] == want[clear | ties]).all())
    if nt > 1:
        assert bool((got[ties] == 0).all()) and int(ties.sum()) >= 4 * w
    assert float((~clear & ~ties).double().mean()) < 0.01
    npp = torch.softmax(logits[1], -1)[..., 1]
    assert float((out[..., 1].double() - npp).abs().max()) <= 1e-6
    hv = logits[2]
    S = torch.einsum("bhwc,oc->bhwo", feats[2].value().abs(), ws[2].double().abs()) + bs[2].double().abs()
    assert bool(((out[..., 2:].double() - hv).abs() <= 66 * U * S).all())
    assert all(f.canaries_intact() for f in feats)


# ------------------------------------------------------------------------------------------------ k. range guard
EDGE = [(65504.0, 0), (float(np.nextafter(np.float32(65504), np.float32(np.inf))), 1), (float("inf"), 1),
        (float("-inf"), 1), (float("nan"), 1)]


def _conv_range(L, prec, path, site, v, trunc=1):
    """Flag raised by one convolution whose stored outputs are all v.  plain: a 1x1 conv of a one-hot input with unit
    weights gives raw = 1 exactly, and BN scale 0 / shift v (relu = 0) makes t = v.  up2: a zero input and skip = v.
    xf: the transform forms relu(0 * 0 + v) from a zero raw tensor."""
    one = prec == "high"
    B, h, w, c, cout = 1, 4, 4, 64, 64
    d = [0] * 80
    d[70], d[72], d[75], d[76], d[77] = 1, 1, B, h, w
    keep = []
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    vec = lambda val, n=cout: torch.full((n,), val, dtype=torch.float32, device="cuda")  # noqa: E731
    A = Split(B, h, w, c, one)
    keep.append(A)
    d[0:8] = A.desc()
    if site == "xf":
        R = Raw(B, h, w, c)
        R.p.zero_()
        sc, sh = vec(0.0, c), vec(v, c)
        keep += [R, sc, sh]
        d[8:16], d[65], d[66] = R.desc(), sc.data_ptr(), sh.data_ptr()
    else:
        x = torch.zeros(B, h, w, c)
        if site == "plain":
            x[..., 0] = 1
        A.fill(*[t.cuda() for t in split_host(x)]) if not one else A.fill(x.half().cuda())
    wt = torch.zeros(cout, c, 1, 1)
    wt[:, 0] = 1.0
    whi, wlo, osc, _ = weight_planes(wt, one)
    keep += [whi, wlo, osc]
    d[56], d[57], d[58] = whi.data_ptr(), 0 if wlo is None else wlo.data_ptr(), osc.data_ptr()
    d[59], d[60], d[61], d[62], d[63], d[64] = 1, cout, c, 64, 1, 1
    if site == "up2":
        SK = Split(B, 2 * h, 2 * w, cout, one)
        sv = torch.full((B, 2 * h, 2 * w, cout), v)
        SK.fill(sv.half().cuda()) if one else SK.fill(*[t.cuda() for t in split_host(sv)])
        OS = Split(B, 2 * h, 2 * w, cout, one)
        keep += [SK, OS]
        d[48:56], d[40:48], d[79] = SK.desc(), OS.desc(), 1
    else:
        OS = Split(B, h, w, cout, one)
        sc_b, sh_b = (vec(1.0), vec(0.0)) if site == "xf" else (vec(0.0), vec(v))
        keep += [OS, sc_b, sh_b]
        d[40:48], d[67], d[68] = OS.desc(), sc_b.data_ptr(), sh_b.data_ptr()
    d[69] = flag.data_ptr()
    info = (ctypes.c_int * 10)()
    L.probe_set_knobs(0, 4, 4, trunc)
    try:
        torch.cuda.synchronize()
        rc = L.probe_conv(_i64(d), 0 if path == "tc" else 1, info)
    finally:
        L.probe_set_knobs(*DEFAULT_KNOBS)
    assert rc == 0
    return int(flag.item())


@pytest.mark.parametrize("site", ["plain", "up2", "xf"])
def test_range_guard_conv(probe, site):
    """65504 is in range; the next fp32 value, +-Inf and NaN raise the flag.  The XF transform applies a ReLU first, so
    -Inf is in range there (relu(-inf) = 0) and NaN raises it from the transform's running maximum -- except with the
    truncating split, whose lo plane of -Inf is -inf - (-inf) = NaN: that layer's output is NaN and its store raises
    the flag instead of returning a clamped value."""
    for prec in PRECS:
        for path in PATHS:
            for trunc in ((1, 0) if site == "xf" and path == "tc" and prec == "highest" else (1,)):
                for v, want in EDGE:
                    if site == "xf" and v == float("-inf"):
                        want = int(trunc == 1 and path == "tc" and prec == "highest")
                    if site == "up2" and prec == "high" and v != 65504.0 and math.isfinite(v):
                        continue                                # a single fp16 skip plane cannot hold it
                    got = _conv_range(probe, prec, path, site, v, trunc)
                    assert got == want, "%s %s %s trunc=%d v=%r: flag %d, expected %d" % (
                        site, prec, path, trunc, v, got, want)


def test_range_guard_elementwise_and_stems(probe):
    B, h, w, c = 1, 4, 4, 64
    for prec in PRECS:
        one = prec == "high"
        for v, want in EDGE:
            # k_bnrelu: t = relu(0 * 0 + v); -inf relus to 0 (in range), NaN raises the flag before the ReLU
            R = Raw(B, h, w, c)
            R.p.zero_()
            O = Split(B, h, w, c, one)
            flag = torch.zeros(1, dtype=torch.int32, device="cuda")
            sc, sh = torch.zeros(c, device="cuda"), torch.full((c,), v, device="cuda")
            torch.cuda.synchronize()
            assert probe.probe_bnrelu(_i64(R.desc()), B, sc.data_ptr(), sh.data_ptr(), _i64(O.desc()), flag.data_ptr()) == 0
            assert int(flag.item()) == (0 if v == float("-inf") else want), ("bnrelu", prec, v)
            # k_up2_add: in = v, skip = 0
            R2 = Raw(B, h, w, c)
            R2.p.fill_(v)
            SK = Split(B, 2 * h, 2 * w, c, one)
            SK.hi.zero_()
            if SK.lo is not None:
                SK.lo.zero_()
            O2 = Split(B, 2 * h, 2 * w, c, one)
            flag.zero_()
            torch.cuda.synchronize()
            assert probe.probe_up2_add(_i64(R2.desc()), B, _i64(SK.desc()), _i64(O2.desc()), flag.data_ptr()) == 0
            assert int(flag.item()) == want, ("up2_add", prec, v)
            # stems on a black image: t = relu(0 * scale + v)
            img = torch.zeros(1, 128, 128, 3, dtype=torch.uint8, device="cuda")
            ph, pl, osc, _, core_w, _ = _stem_weights(torch.randn(64, 3, 7, 7), one)
            s0, b0 = torch.ones(64, device="cuda"), torch.full((64,), v, device="cuda")
            for path in (0, 1):
                OS = Split(1, 128, 128, 64, one)
                flag.zero_()
                torch.cuda.synchronize()
                rc = probe.probe_conv0(img.data_ptr(), 1, 128, 128, 3, path, ph.data_ptr(), 0 if pl is None else pl.data_ptr(),
                                       osc.data_ptr(), core_w.data_ptr(), s0.data_ptr(), b0.data_ptr(), _i64(OS.desc()),
                                       flag.data_ptr())
                assert rc == 0
                # ReLU precedes the store: -inf and NaN become 0 (fmaxf), in range
                exp = 0 if v == float("-inf") or v != v else want
                assert int(flag.item()) == exp, ("stem", path, prec, v)


# ------------------------------------------------------------------------------------------------ 3. network self-test
def _fp64_forward_check(net, x, sd, mode, nt):
    from oracle import hovernet_torch as O
    from hover_net_b200.models.hovernet.run_desc import infer_step
    out = infer_step(x, net)
    ref = O.infer_step(x, O.to_torch_state_dict(sd), mode, nt, dtype=torch.float64)
    np_err = np.abs(out[..., -3] - ref[..., -3]).max()
    hv_scale = max(1.0, float(np.abs(ref[..., -2:]).max()))
    hv_err = np.abs(out[..., -2:] - ref[..., -2:]).max() / hv_scale
    assert np_err <= 1e-4 and hv_err <= 1e-4, (np_err, hv_err)


LINE = re.compile(r"^(\S+)\s.*\| raw diff (\S+) \(ref (\S+)\) \| split diff (\S+) \(ref (\S+)\)(.*)$")


def _expected_layers(mode, nt, fuse_shortcut):
    from hover_net_b200 import arch
    names = set()
    for k, v in arch.state_dict_spec(mode, nt).items():
        if len(v) != 4 or k == "conv0./.weight" or ".u0.conv." in k:
            continue
        if fuse_shortcut and k.endswith(".shortcut.weight"):
            continue
        if fuse_shortcut and k.endswith(".units.0.conv3.weight"):
            k = k[: -len(".weight")] + "+shortcut"
        names.add(k)
    return names


@pytest.mark.parametrize("mode,nt,size,B,opts", [
    ("fast", 6, 256, 2, {}),
    ("fast", 6, 272, 1, {}),
    ("original", 5, 278, 3, {"chunk": 2}),
    ("fast", 6, 256, 1, {"fuse_shortcut": 0}),
    ("fast", 6, 256, 1, {"fuse_up2": 0}),
    ("original", None, 270, 1, {"branch_streams": 0}),
], ids=["fast256", "fast272", "orig278_chunk2", "no_fuse_shortcut", "no_fuse_up2", "no_branch_streams"])
@pytest.mark.parametrize("prec", PRECS)
def test_network_selftest(mode, nt, size, B, opts, prec):
    """conv_path=2 runs every wgmma layer next to the CUDA-core referee over the whole tensor: a loose net for indexing
    errors (2^-12 of max(|ref|, 1); 2^-10 for the single-plane split outputs of "high"); the precise per-operator
    bounds are the tests above."""
    from hover_net_b200 import synth
    from hover_net_b200.models.hovernet.net_desc import create_model
    from hover_net_b200.models.hovernet.run_desc import infer_step
    sd = synth.make_state_dict(mode, nt, seed=1)
    net = create_model(mode=mode, input_ch=3, nr_types=nt, precision=prec)
    net.load_state_dict(sd, strict=True)
    for k, v in opts.items():
        net.ctx.set_option(k, v)
    net.ctx.set_option("conv_path", 2)
    x = synth.make_patches(B, size, seed=size + B)
    # a single fp16 plane: the two kernels sum in different orders, and a stored value one rounding boundary apart
    # differs by one fp16 ulp, up to 2^-10 of the tensor's largest value
    split_tol = 2.0 ** -12 if prec == "highest" else 2.0 ** -10
    try:
        out = infer_step(x, net)
        log = net.ctx.debug_log()
    finally:
        net.ctx.set_option("conv_path", 0)
    assert np.isfinite(out).all()
    seen = set()
    for line in log.splitlines():
        m = LINE.match(line)
        assert m, "unparsed self-test line: %r" % line
        name, rd, rr, sd_, sr, tail = m.groups()
        assert "CUDA ERROR" not in tail, line
        rd, rr, sd_, sr = (float(t) for t in (rd, rr, sd_, sr))
        assert max(rd, sd_) < 1e38, "NaN sentinel: %s" % line
        assert rd <= 2.0 ** -12 * max(rr, 1.0) and sd_ <= split_tol * max(sr, 1.0), line
        seen.add(name)
    assert seen == _expected_layers(mode, nt, opts.get("fuse_shortcut", 1)), sorted(seen ^ _expected_layers(mode, nt, opts.get("fuse_shortcut", 1)))
    if prec == "highest" and size in (272, 278):
        _fp64_forward_check(net, x[:1], sd, mode, nt)
    net.ctx.close()


# ------------------------------------------------------------------------------------------------ 4. finalize
@pytest.mark.parametrize("key,val", [
    ("d1.units.1.conv1/bn.weight", float("nan")), ("conv0.bn.bias", float("inf")),
    ("decoder.np.u2.dense.units.0.preact_bna/bn.running_mean", float("-inf")),
    ("d0.blk_bna.bn.running_var", -1.0), ("d2.units.0.conv2/bn.running_var", -2e-5),
    ("decoder.hv.u0.conv.weight", float("nan")), ("decoder.tp.u0.conv.bias", float("inf")),
])
def test_finalize_rejects_non_finite_parameters(key, val):
    from hover_net_b200 import _lib, synth
    from hover_net_b200.models.hovernet.net_desc import create_model
    sd = dict(synth.make_state_dict("fast", 6, seed=0))
    a = np.array(sd[key], dtype=np.float32, copy=True)
    a.flat[a.size // 2] = val
    sd[key] = a
    net = create_model(mode="fast", input_ch=3, nr_types=6)
    with pytest.raises(_lib.HvnError) as e:
        net.load_state_dict(sd, strict=True)
    assert e.value.code == -3 and key in str(e.value)
    net.ctx.close()


# ------------------------------------------------------------------------------------------------ a. coverage (last)
def test_instantiation_coverage():
    """Every reachable k_conv_tc instantiation ran above: (BLOCK_N, epilogue, XF, ONE) = 18 without XF plus
    XF x {64, 128} x {PLAIN, UP2} x ONE."""
    want = {(bn, e, 0, o) for bn in (32, 64, 128) for e in (0, 1, 2) for o in (0, 1)}
    want |= {(bn, e, 1, o) for bn in (64, 128) for e in (0, 2) for o in (0, 1)}
    assert len(want) == 26
    for path in PATHS:
        for prec in PRECS:  # XF layers also carry their operand's rounding, outside gamma: reported apart
            for xf in (False, True):
                r = [x for x in RATIOS if x[2:] == (path, prec, xf)]
                if r:
                    w = max(r, key=lambda x: x[0] / x[1])
                    print("  %-4s %-7s %s worst raw err/(S*2^-24) = %.2f against gamma/2^-24 = %.1f (%d cases)" % (
                        path, prec, "XF" if xf else "  ", w[0], w[1], len(r)))
    print("  dispatched %d instantiations" % len(DISPATCHED))
    assert DISPATCHED == want, "missing %s" % sorted(want - DISPATCHED)
