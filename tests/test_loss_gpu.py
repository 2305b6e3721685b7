"""The validation loss on the H100 (hvn_valid_loss*, k_loss_reduce, k_head_full, k_tta_merge_full).

* The reduction alone, through tests/native/libhvn_loss_probe.so (the product's own loss.o), on the recorded cases of
  the reference's loss functions (tests/golden/loss_cases.npz) embedded in larger maps: within 1e-5 |ref| + 1e-7 of
  the reference's losses, within 1e-6 |ref| + 1e-9 of the float64 restatement (tests/loss_ref.py) slot by slot, and
  bit-identical from call to call.  The reference itself only runs where the goldens are generated; loss_ref.py is
  checked against it there (tests/test_loss_cpu.py) and stands in for it here.
* End to end: sums against loss_ref.py applied to the returned probabilities and the device's own targets; counts,
  hv_sse and flags against hvn_valid; the plain forward untouched; determinism over calls and chunk sizes; both
  precisions, TTA on and off, both modes, nr_types None / 5 / 6.
* The errors: an out-of-range type id inside the crop, and the range error."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from hover_net_b200 import arch, synth
from hover_net_b200.models.hovernet import run_desc

import loss_ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "loss_cases.npz")


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def probe():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("no CUDA device")
    sys.path.insert(0, os.path.join(ROOT, "tests", "native"))
    try:
        import build_loss_probe
    finally:
        sys.path.pop(0)
    L = ctypes.CDLL(build_loss_probe.build())
    ll = ctypes.c_longlong
    L.loss_probe_reduce.argtypes = [ll, ll, ll, ll] + [ctypes.c_int] * 6 + [ll, ll, ctypes.POINTER(ctypes.c_int)]
    L.loss_probe_nsums.argtypes = [ctypes.c_int]
    yield L
    L.loss_probe_release()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _probe_reduce(L, probs, inst, typ, hv, h, w, nt):
    import torch
    B, H, W = inst.shape
    sums = torch.full((L.loss_probe_nsums(nt),), np.nan, dtype=torch.float64, device="cuda")
    counts = torch.zeros((3 + 2 * nt,), dtype=torch.int64, device="cuda")
    bad = ctypes.c_int(-1)
    d = [_dev(probs), _dev(inst), _dev(typ) if typ is not None else None, _dev(hv)]
    rc = L.loss_probe_reduce(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr() if d[2] is not None else 0,
                             d[3].data_ptr(), B, H, W, h, w, nt, sums.data_ptr(), counts.data_ptr(), ctypes.byref(bad))
    assert rc == 0, rc
    return sums.cpu().numpy(), counts.cpu().numpy(), bad.value


def _embed(rng, crop, pad, fill):
    """crop [B,h,w,...] into a [B,h+pad,w+pad,...] map at cropping_center's offset, the border filled by fill()."""
    B, h, w = crop.shape[:3]
    out = fill((B, h + pad[0], w + pad[1]) + crop.shape[3:]).astype(crop.dtype)
    y0, x0 = int(pad[0] * 0.5), int(pad[1] * 0.5)
    out[:, y0:y0 + h, x0:x0 + w] = crop
    return out


def _host_counts(probs, fg, tp, nt):
    pn, tn = probs[..., 1] > np.float32(0.5), fg > 0
    c = [int((pn == tn).sum()), int((pn & tn).sum()), int(pn.sum() + tn.sum())]
    if nt:
        pt = np.argmax(probs[..., 4:], -1)  # first maximal index, k_head's rule
        for k in range(nt):
            pk, tk = pt == k, tp == k
            c += [int((pk & tk).sum()), int(pk.sum() + tk.sum())]
    return np.array(c, np.int64)


def _check_sums(got, want, what):
    assert got.shape == want.shape, what
    err = np.abs(got - want)
    assert (err <= 1e-6 * np.abs(want) + 1e-9).all(), (what, np.flatnonzero(err > 1e-6 * np.abs(want) + 1e-9),
                                                       got, want)


def test_kernel_on_reference_cases(probe):
    g = np.load(GOLDEN)
    res = json.loads(str(g["results"]))
    rng = np.random.default_rng(5)
    for name, r in res.items():
        nt = r["nt"]
        probs, fg, hv = g["probs_" + name], g["fg_" + name], g["hv_" + name]
        tp = g["tp_" + name] if nt else None
        B, h, w = fg.shape
        pad = (7, 5)
        # outside the crop: instances, HV noise and type ids no map may hold; none of it may be read
        inst = _embed(rng, fg.astype(np.int32) * rng.integers(1, 50, fg.shape).astype(np.int32), pad,
                      lambda s: rng.integers(0, 9, s))
        hvf = _embed(rng, hv, pad, lambda s: rng.normal(0, 3, s))
        typ = _embed(rng, tp, pad, lambda s: np.full(s, 99)) if nt else None
        sums, counts, bad = _probe_reduce(probe, probs, inst, typ, hvf, h, w, nt)
        assert bad == 0, name
        _check_sums(sums, loss_ref.sums(probs, fg, hv, tp), name)
        got = run_desc.loss_scalars(sums, fg.size)
        for k, v in got.items():
            assert abs(v - r[k]) <= 1e-5 * abs(r[k]) + 1e-7, (name, k, v, r[k])
        assert np.array_equal(counts, _host_counts(probs, fg, tp, nt)), name
        again, _, _ = _probe_reduce(probe, probs, inst, typ, hvf, h, w, nt)
        assert again.tobytes() == sums.tobytes(), name
        print("%-12s B=%-2d %3dx%-3d nt=%d  max rel err vs fp64 %.2e" % (
            name, B, h, w, nt, float(np.max(np.abs(sums - loss_ref.sums(probs, fg, hv, tp)) /
                                           np.maximum(np.abs(loss_ref.sums(probs, fg, hv, tp)), 1e-300)))))


def test_kernel_flags_out_of_range_types_in_the_crop_only(probe):
    g = np.load(GOLDEN)
    probs, fg, hv, tp = (g[k + "_c3x3_t5"] for k in ("probs", "fg", "hv", "tp"))
    for bad_id in (5, -1):
        t = tp.copy()
        t[2, 1, 2] = bad_id
        _, _, bad = _probe_reduce(probe, probs, fg.astype(np.int32), t, hv, 3, 3, 5)
        assert bad == 1, bad_id


# ------------------------------------------------------------------------------------------------ end to end
def _net(mode, nt, precision="highest", tta=False, sd=None):
    from hover_net_b200.models.hovernet.net_desc import create_model
    net = create_model(mode=mode, input_ch=3, nr_types=nt, precision=precision, tta=tta)
    net.load_state_dict(sd if sd is not None else synth.make_state_dict(mode, nt, seed=0), strict=True)
    return net


def _batch(mode, nt, B, seed):
    size = arch.PATCH_GEOMETRY[mode][0]
    imgs = synth.make_patches(B, size, seed=seed)
    inst = np.stack([synth.synth_instances(size, size, seed=seed * 10 + i) for i in range(B)])
    typ = np.where(inst > 0, inst % nt, 0).astype(np.int32) if nt else None
    return imgs, inst, typ


def _crop(a, h, w):
    H, W = a.shape[1:3]
    y0, x0 = int((H - h) * 0.5), int((W - w) * 0.5)
    return a[:, y0:y0 + h, x0:x0 + w]


@pytest.mark.parametrize("tta", [False, True])
@pytest.mark.parametrize("precision", ["highest", "high"])
@pytest.mark.parametrize("mode,nt", [("original", None), ("original", 5), ("fast", 6)])
def test_valid_loss_end_to_end(mode, nt, precision, tta):
    B = 3
    imgs, inst, typ = _batch(mode, nt, B, seed=31)
    net = _net(mode, nt, precision, tta)
    ctx = net.ctx
    try:
        plain0 = ctx.forward(imgs)
        counts, sse, flags, sums, probs = ctx.valid_loss(imgs, inst, typ, want_probs=True)
        plain1 = ctx.forward(imgs)
        assert plain0.tobytes() == plain1.tobytes(), "a loss call changed the plain forward"
        h, w = plain0.shape[1:3]
        ntt = nt or 0
        assert probs.shape == (B, h, w, 4 + ntt) and sums.shape == (10 + (1 + 3 * ntt if nt else 0),)
        # the probabilities agree with the plain forward: NP p1 and HV bit for bit, TP through k_head's argmax rule
        assert np.array_equal(_bits(probs[..., 1]), _bits(plain0[..., -3]))
        assert np.array_equal(_bits(probs[..., 2:4]), _bits(plain0[..., -2:]))
        if nt:
            assert np.array_equal(np.argmax(probs[..., 4:], -1).astype(np.float32), plain0[..., 0])
        # counts, hv_sse and flags: hvn_valid's
        c2, s2, f2 = ctx.valid(imgs, inst, typ)
        assert np.array_equal(counts, c2) and np.array_equal(flags, f2)
        assert abs(sse - s2) <= 1e-12 * s2 and sse == sums[7]
        # the sums: the fp64 restatement on the returned probabilities and the device's own targets
        hv_full, _ = ctx.targets(inst, (h, w))
        fg_c, hv_c = _crop(inst, h, w) > 0, _crop(hv_full, h, w)
        tp_c = _crop(typ, h, w) if nt else None
        _check_sums(sums, loss_ref.sums(probs, fg_c, hv_c, tp_c), (mode, nt, precision, tta))
        scal = run_desc.loss_scalars(sums, fg_c.size)
        assert all(np.isfinite(v) for v in scal.values())
        # deterministic: again, and with another chunk size
        for chunk in (32, 12):
            ctx.set_option("chunk", chunk)
            again = ctx.valid_loss(imgs, inst, typ)[3]
            assert again.tobytes() == sums.tobytes(), chunk
        print("\n%s/%s %s tta=%d: %s" % (mode, nt, precision, tta, " ".join("%s=%.6g" % kv for kv in scal.items())))
    finally:
        ctx.close()


def test_valid_loss_device_pointers():
    mode, nt = "original", 5
    imgs, inst, typ = _batch(mode, nt, 2, seed=33)
    net = _net(mode, nt)
    ctx = net.ctx
    counts, sse, flags, sums, probs = ctx.valid_loss(imgs, inst, typ, want_probs=True)
    B, H, W = inst.shape
    nc, ns = counts.size, sums.size
    d = [ctx.malloc(n) for n in (imgs.nbytes, inst.nbytes, typ.nbytes, nc * 8, 8, B * 4, ns * 8, probs.nbytes)]
    try:
        ctx.h2d(d[0], imgs, imgs.nbytes)
        ctx.h2d(d[1], inst, inst.nbytes)
        ctx.h2d(d[2], typ, typ.nbytes)
        for want_probs in (True, False):
            ctx.valid_loss_dev(d[0], d[1], d[2], B, H, W, d[3], d[4], d[5], d[6], d[7] if want_probs else None)
            c2, s2, f2 = np.zeros(nc, np.int64), np.zeros(1), np.zeros(B, np.int32)
            m2, p2 = np.zeros(ns), np.zeros_like(probs)
            for a, p in ((c2, d[3]), (s2, d[4]), (f2, d[5]), (m2, d[6]), (p2, d[7])):
                ctx.d2h(a, p, a.nbytes)
            assert np.array_equal(c2, counts) and s2[0] == sse and np.array_equal(f2, flags)
            assert m2.tobytes() == sums.tobytes() and p2.tobytes() == probs.tobytes()
        ctx.set_option("profile", 1)
        ctx.valid_loss_dev(d[0], d[1], d[2], B, H, W, d[3], d[4], d[5], d[6], None)
        assert ctx.stage_ms("loss") > 0.0
    finally:
        for p in d:
            ctx.free(p)
        ctx.close()


def test_out_of_range_type_is_invalid():
    from hover_net_b200._lib import HvnError
    mode, nt = "original", 5
    imgs, inst, typ = _batch(mode, nt, 2, seed=35)
    net = _net(mode, nt)
    try:
        for bad_id in (nt, -3):
            bad = typ.copy()
            bad[1, 135, 140] = bad_id  # inside the 80 x 80 crop (rows / cols 95..174)
            with pytest.raises(HvnError) as e:
                net.ctx.valid_loss(imgs, inst, bad)
            assert e.value.code == -1 and "type id" in str(e.value)
            net.ctx.valid(imgs, inst, bad)  # hvn_valid keeps ignoring such ids
        outside = typ.copy()
        outside[0, 3, 3] = 77  # outside the crop: not part of the loss
        a = net.ctx.valid_loss(imgs, inst, outside)[3]
        b = net.ctx.valid_loss(imgs, inst, typ)[3]
        assert a.tobytes() == b.tobytes()
        with pytest.raises(HvnError):
            net.ctx.valid_loss(imgs, inst, None)  # a typed model needs the type map
    finally:
        net.ctx.close()


def test_range_error_as_in_valid():
    """Activations past the fp16-split range: the raw entry point returns HVN_ERR_RANGE, the binding retries with a
    higher act_shift, and the result then matches hvn_valid's on the same context."""
    from hover_net_b200 import _lib
    mode, nt = "fast", 6
    sd = dict(synth.make_state_dict(mode, nt, seed=0))
    sd["conv0./.weight"] = (sd["conv0./.weight"] * np.float32(3.0e5)).astype(np.float32)
    sd["conv0.bn.running_var"] = np.full_like(sd["conv0.bn.running_var"], 1.0)
    net = _net(mode, nt, sd=sd)
    imgs, inst, typ = _batch(mode, nt, 1, seed=37)
    try:
        L = _lib.lib()
        L.hvn_valid_loss.argtypes = net.ctx._VALID_LOSS_ARGS
        counts, sse = np.zeros(3 + 2 * nt, np.int64), np.zeros(1)
        flags, sums = np.zeros(1, np.int32), np.zeros(11 + 3 * nt)
        p = _lib._ptr
        rc = L.hvn_valid_loss(net.ctx._h, p(imgs), p(inst), p(typ), 1, 256, 256, p(counts), p(sse), p(flags),
                              p(sums), None)
        assert rc == -6 and b"act_shift" in L.hvn_last_error()
        c, s, f, sm, _ = net.ctx.valid_loss(imgs, inst, typ)
        assert net.ctx.counter("act_shift") > 0 and np.isfinite(sm).all()
        c2, s2, _ = net.ctx.valid(imgs, inst, typ)
        assert np.array_equal(c, c2) and abs(s - s2) <= 1e-12 * s2
    finally:
        net.ctx.close()


def test_run_valid_loss_end_to_end(tmp_path):
    from test_oracle_targets import _write_patches
    mode, nt = "original", 5
    _write_patches(tmp_path, 5, 300, True, seed=3)
    ck = tmp_path / "ck.npz"
    np.savez(ck, **{k: np.asarray(v) for k, v in synth.make_state_dict(mode, nt, seed=0).items()})
    outs = {}
    for tag, extra in (("plain", []), ("loss2", ["--loss", "--batch_size", "2"]), ("loss5", ["--loss", "--batch_size", "5"])):
        out = tmp_path / (tag + ".json")
        r = subprocess.run([sys.executable, "-m", "hover_net_b200.run_valid", "--model_path", str(ck), "--valid_dir",
                            str(tmp_path), "--nr_types", str(nt), "--json", str(out)] + extra,
                           cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        outs[tag] = (r.stdout, json.loads(out.read_text()))
    plain, loss2, loss5 = (outs[k][1] for k in ("plain", "loss2", "loss5"))
    names = ["loss_tp_bce", "loss_tp_dice", "loss_np_bce", "loss_np_dice", "loss_hv_mse", "loss_hv_msge",
             "overall_loss"]
    assert list(loss2) == list(plain) + names
    for k in plain:
        if k == "hv_mse":
            assert abs(loss2[k] - plain[k]) <= 1e-12 * plain[k]
        else:
            assert loss2[k] == plain[k], k
    for k in names:  # the set's loss does not depend on the batch size
        assert abs(loss2[k] - loss5[k]) <= 1e-12 * abs(loss5[k]), k
    printed = dict(line.split(": ") for line in outs["loss2"][0].strip().split("\n"))
    assert {k: float(v) for k, v in printed.items()} == loss2
