"""CPU checks of the host restatements the operator tests (test_conv_kernels_gpu.py) build their references from: the
fp16 split, the TF-"same" padding rule, the weight planes and the fp64 convolution."""
import numpy as np
import torch

from test_conv_kernels_gpu import conv64, split_host, tf_same_lo, values, weight_planes


def test_split_matches_fp16_rounding():
    g = torch.Generator().manual_seed(0)
    x = torch.cat([values((4096,), "wide", g), values((4096,), "normal", g), values((1024,), "coherent", g),
                   torch.tensor([0.0, -0.0, 65504.0, -65504.0, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26, 1 + 2.0 ** -11])])
    hi, lo = split_host(x)
    xn = x.numpy()
    hn = xn.astype(np.float16)                       # IEEE round-to-nearest-even, independent of torch
    assert np.array_equal(hi.numpy().view(np.uint16), hn.view(np.uint16))
    rn = (xn - hn.astype(np.float32)).astype(np.float16)
    assert np.array_equal(lo.numpy().view(np.uint16), rn.view(np.uint16))
    # hi + lo carries x to 2^-22 relative, plus half the smallest fp16 subnormal where lo (or hi) is subnormal
    m = np.abs(xn) <= 65504
    err = np.abs(hn[m].astype(np.float64) + rn[m].astype(np.float64) - xn[m])
    assert (err <= 2.0 ** -22 * np.abs(xn[m]) + 2.0 ** -25).all()
    # the coherent operands: lo about 2^-11 of |x| and positive
    hc, lc = split_host(values((1000,), "coherent", g))
    r = lc.double() / hc.double()
    assert bool((r > 2.0 ** -11.4).all()) and bool((r < 2.0 ** -10.9).all())


def test_tf_same_padding_rule():
    """net_utils.py's TF-"same" rule as cnn.cu restates it: total pad = max(k - s, 0) if size % s == 0 else
    max(k - size % s, 0), the smaller half above / left; the output size is ceil(size / s)."""
    assert tf_same_lo(16, 3, 2) == 0 and tf_same_lo(15, 3, 2) == 1
    assert tf_same_lo(64, 3, 1) == 1 and tf_same_lo(7, 3, 1) == 1 and tf_same_lo(9, 1, 2) == 0
    for size in range(1, 40):
        for k in (1, 3, 5):
            for s in (1, 2):
                lo = tf_same_lo(size, k, s)
                total = max(k - s, 0) if size % s == 0 else max(k - size % s, 0)
                out = -(-size // s)
                assert lo == total // 2 and (out - 1) * s + k <= size + total


def test_weight_planes_restate_make_conv():
    g = torch.Generator().manual_seed(1)
    w = values((8, 70, 3, 3), "normal", g) * torch.pow(2.0, torch.arange(-8, 8, 2).float()).view(8, 1, 1, 1)
    w[3] = 0
    hi, lo, osc, st = (t.cpu() if t is not None else None for t in weight_planes(w, False, "cpu"))
    assert hi.shape == (9, 8, 128) and bool((hi[:, :, 70:] == 0).all())
    mx = (hi.float().abs().amax(dim=(0, 2)))
    nz = torch.arange(8) != 3
    assert bool((mx[nz] >= 2.0 ** 13).all()) and bool((mx[nz] < 2.0 ** 14).all()) and float(osc[3]) == 1.0
    # 22 bits per weight, down to half an fp16 subnormal of the channel's scaled planes
    assert bool(((st - w.double()).abs() <= 2.0 ** -22 * w.double().abs() + 2.0 ** -25 * osc.double().view(8, 1, 1, 1)).all())
    hi1, lo1, _, st1 = weight_planes(w, True, "cpu")
    assert lo1 is None and torch.equal(hi1.cpu(), hi)


def test_conv64_against_a_direct_loop():
    g = torch.Generator().manual_seed(2)
    for (B, h, w, c, o, k, s, pad) in [(2, 5, 6, 3, 4, 3, 1, 1), (1, 7, 5, 2, 3, 3, 2, 1), (1, 6, 6, 2, 2, 5, 1, 0),
                                       (2, 4, 3, 3, 2, 1, 2, 0)]:
        a = torch.randn(B, h, w, c, generator=g, dtype=torch.float64)
        wt = torch.randn(o, c, k, k, generator=g, dtype=torch.float64)
        ho, wo = -(-(h + 2 * pad - k + 1) // s), -(-(w + 2 * pad - k + 1) // s)
        got = conv64(a, wt, s, pad, ho, wo).numpy()
        ref = np.zeros((B, ho, wo, o))
        an, wn = a.numpy(), wt.numpy()
        for n in range(B):
            for y in range(ho):
                for x in range(wo):
                    for ky in range(k):
                        for kx in range(k):
                            iy, ix = y * s - pad + ky, x * s - pad + kx
                            if 0 <= iy < h and 0 <= ix < w:
                                ref[n, y, x] += wn[:, :, ky, kx] @ an[n, iy, ix]
        assert np.allclose(got, ref, rtol=1e-12, atol=1e-12)
