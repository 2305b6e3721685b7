"""Precision "high" on the H100: accuracy against the reference graph as its users run it on this GPU (PyTorch fp32
with cuDNN TF32 convolutions, the default), robustness, the untouched default, consistency and memory.

Referee for every accuracy number: the fp64 oracle forward on the same checkpoint and patches.  The TF32 arm is the
same oracle in fp32 on the GPU with torch.backends.cudnn.allow_tf32 = True."""
import ctypes

import numpy as np
import pytest
import torch

from hover_net_b200 import arch, synth

pytestmark = pytest.mark.gpu


def _net(mode, nt, sd, precision):
    from hover_net_b200.models.hovernet.net_desc import create_model
    net = create_model(mode=mode, input_ch=3, nr_types=nt, precision=precision)
    net.load_state_dict(sd, strict=True)
    return net


def _oracle(x, sd, mode, nt, dtype):
    from oracle import hovernet_torch as O
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        return O.infer_step(x, O.to_torch_state_dict(sd), mode, nt, dtype=dtype, device="cuda")
    finally:
        torch.backends.cudnn.allow_tf32 = prev


def _errors(out, ref, nt):
    """NP max abs error, HV max abs error relative to the map's scale (as tests/test_cnn_gpu.py), mean abs error over
    NP and HV, TP-argmax mismatch fraction."""
    hv_scale = max(1.0, float(np.abs(ref[..., -2:]).max()))
    return {"np_max": float(np.abs(out[..., -3] - ref[..., -3]).max()),
            "hv_rel": float(np.abs(out[..., -2:] - ref[..., -2:]).max()) / hv_scale,
            "mean": float(np.abs(out[..., -3:] - ref[..., -3:]).mean()),
            "tp": float((out[..., 0] != ref[..., 0]).mean()) if nt else 0.0}


def _assert_within_tf32_bar(out, x, sd, mode, nt, tag):
    """out (precision "high") against the fp64 referee: each error at most twice the TF32 arm's on the same input."""
    ref = _oracle(x, sd, mode, nt, torch.float64)
    tf32 = _oracle(x, sd, mode, nt, torch.float32)
    assert np.isfinite(out).all(), tag
    e_tf, e_hi = _errors(tf32, ref, nt), _errors(out, ref, nt)
    print("\n%s  TF32 arm: %s\n%s  high:     %s" % (tag, e_tf, tag, e_hi))
    for k in ("np_max", "hv_rel", "mean"):
        assert e_hi[k] <= 2.0 * e_tf[k], "%s: %s %.3e > 2 x TF32 arm %.3e" % (tag, k, e_hi[k], e_tf[k])
    assert e_hi["tp"] <= max(2.0 * e_tf["tp"], 2e-3), "%s: tp mismatch %.3e (TF32 arm %.3e)" % (tag, e_hi["tp"], e_tf["tp"])


def _check_vs_tf32(sd, mode, nt, tag, n=2):
    from hover_net_b200.models.hovernet.run_desc import infer_step
    x = synth.make_patches(n, arch.PATCH_GEOMETRY[mode][0], seed=33)
    net = _net(mode, nt, sd, "high")
    out = infer_step(x, net)
    net.ctx.close()
    _assert_within_tf32_bar(out, x, sd, mode, nt, tag)


@pytest.mark.parametrize("mode,nt", [("original", None), ("original", 5), ("fast", 6)])
def test_high_is_as_accurate_as_the_reference_tf32_path(mode, nt):
    _check_vs_tf32(synth.make_state_dict(mode, nt, seed=0), mode, nt, "%s/%s" % (mode, nt))


def test_high_with_layerwise_power_of_two_rescaling():
    """Weights of every BN-fed convolution scaled by 2^+-8 with the BN statistics rescaled to match."""
    mode, nt = "fast", 6
    sd = dict(synth.make_state_dict(mode, nt, seed=0))
    rng = np.random.default_rng(5)
    for k in list(sd):
        if not k.endswith(".weight") or sd[k].ndim != 4:
            continue
        bn = "conv0.bn" if k == "conv0./.weight" else k[: -len(".weight")] + "/bn"
        if bn + ".running_mean" not in sd:
            continue
        e = int(rng.choice([-8, 8]))
        sd[k] = (sd[k] * np.float32(2.0 ** e)).astype(np.float32)
        sd[bn + ".running_mean"] = (sd[bn + ".running_mean"] * np.float32(2.0 ** e)).astype(np.float32)
        sd[bn + ".running_var"] = (sd[bn + ".running_var"] * np.float32(4.0 ** e)).astype(np.float32)
    _check_vs_tf32(sd, mode, nt, "2^+-8 per layer")


def test_high_with_heavy_tailed_weights():
    mode, nt = "original", None
    sd = dict(synth.make_state_dict(mode, nt, seed=0))
    rng = np.random.default_rng(13)
    for k, v in sd.items():
        if v.ndim == 4 and ".u0.conv." not in k:
            t = rng.standard_t(3, v.shape).astype(np.float32)
            sd[k] = (t * (np.std(v) / np.std(t))).astype(np.float32)
    _check_vs_tf32(sd, mode, nt, "student-t weights")


def test_high_reference_weights_init_checkpoint():
    """The reference's own initialisation (Kaiming-normal convolutions, identity BN; HV maps ~1e4): finite through the
    binding (which answers any HVN_ERR_RANGE with an exact act_shift retry) and within the TF32 bar."""
    from hover_net_b200.models.hovernet.run_desc import infer_step
    mode, nt = "fast", 6
    sd = dict(synth.make_state_dict(mode, nt, seed=0))
    rng = np.random.default_rng(11)
    for k, v in sd.items():
        if k.endswith("num_batches_tracked") or k == "upsample2x.unpool_mat":
            continue
        if v.ndim == 4:
            o, i, kh, kw = v.shape
            sd[k] = (np.sqrt(2.0 / (o * kh * kw)) * rng.standard_normal(v.shape)).astype(np.float32)
        elif k.endswith("running_mean") or k.endswith(".bias"):
            sd[k] = np.zeros_like(v)
        else:
            sd[k] = np.ones_like(v)
    x = synth.make_patches(1, 256, seed=33)
    net = _net(mode, nt, sd, "high")
    out = infer_step(x, net)
    print("\nweights_init, high: act_shift after the call %d" % net.ctx.counter("act_shift"))
    net.ctx.close()
    _assert_within_tf32_bar(out, x, sd, mode, nt, "weights_init")


def test_high_range_overflow_is_an_error_then_retry():
    """Stem activations pushed past 65504: HVN_ERR_RANGE through the raw C ABI in "high" mode, then the binding's
    act_shift retry returns a finite map."""
    from hover_net_b200 import _lib
    from hover_net_b200.models.hovernet.run_desc import infer_step
    mode, nt = "fast", 6
    sd = dict(synth.make_state_dict(mode, nt, seed=0))
    sd["conv0./.weight"] = (sd["conv0./.weight"] * np.float32(3.0e5)).astype(np.float32)
    sd["conv0.bn.running_var"] = np.full_like(sd["conv0.bn.running_var"], 1.0)
    net = _net(mode, nt, sd, "high")
    x = synth.make_patches(1, 256, seed=3)
    out = np.empty((1, 164, 164, 4), np.float32)
    L = _lib.lib()
    rc = L.hvn_forward(net.ctx._h, x.ctypes.data_as(ctypes.c_void_p), 1, 256, 256, out.ctypes.data_as(ctypes.c_void_p))
    assert rc == -6 and b"act_shift" in L.hvn_last_error()
    out = infer_step(x, net)
    assert np.isfinite(out).all() and net.ctx.counter("act_shift") > 0 and net.ctx.counter("precision") == 1
    net.ctx.close()


def test_default_is_untouched_by_switching():
    from hover_net_b200.models.hovernet.run_desc import infer_step
    from hover_net_b200._lib import HvnError
    mode, nt = "original", 5
    sd = synth.make_state_dict(mode, nt, seed=0)
    x = synth.make_patches(2, 270, seed=23)
    fresh = _net(mode, nt, sd, "highest")
    a = infer_step(x, fresh)
    assert fresh.ctx.counter("precision") == 0
    fresh.ctx.set_option("precision", 0)   # explicit default: nothing changes
    assert np.array_equal(infer_step(x, fresh), a)
    with pytest.raises(HvnError):
        fresh.ctx.set_option("precision", 2)
    fresh.ctx.close()
    sw = _net(mode, nt, sd, "highest")
    sw.ctx.set_option("precision", 1)
    h = infer_step(x, sw)
    assert sw.ctx.counter("precision") == 1 and not np.array_equal(h, a)
    sw.ctx.set_option("precision", 0)
    assert np.array_equal(infer_step(x, sw), a), "highest -> high -> highest must reproduce highest bit for bit"
    sw.ctx.close()


def test_high_is_self_consistent():
    from hover_net_b200.models.hovernet.post_proc import process
    from hover_net_b200.models.hovernet.run_desc import infer_step, infer_step_fused
    mode, nt = "fast", 6
    net = _net(mode, nt, synth.make_state_dict(mode, nt, seed=0), "high")
    x = synth.make_patches(3, 256, seed=21)
    a = infer_step(x, net)
    assert np.array_equal(infer_step(x, net), a), "two runs"
    net.ctx.set_option("chunk", 2)
    c2 = infer_step(x, net)
    net.ctx.set_option("chunk", 3)
    assert np.array_equal(infer_step(x, net), c2), "chunk 2 vs chunk 3"
    net.ctx.set_option("chunk", 0)
    pred = infer_step(x[:2], net)
    fpred, finst, _, _ = infer_step_fused(x[:2], net)
    assert np.array_equal(pred, fpred)
    for i in range(2):
        inst, _ = process(pred[i], nr_types=nt, return_centroids=True)
        assert np.array_equal(inst, finst[i]), "fused vs infer_step + process"
    img = np.concatenate([x[0], x[1][:, ::-1]], 1)[:220, :300]
    tp, ti, tt, _, _ = net.ctx.infer_tile(img, 256, 4)
    pi, ptab, pn = net.ctx.postproc(tp, nt)
    assert np.array_equal(ti, pi[0]) and np.array_equal(tt, ptab[0, : int(pn[0])]), "infer_tile vs process(pred)"
    net.ctx.close()


@pytest.mark.parametrize("mode,nt", [("original", 5), ("fast", 6)])
def test_high_kernel_variants_agree(mode, nt):
    """Separate BN+ReLU pass and no L2 prefetch against the default knobs in "high" mode: the same products in the same
    order, so within 3e-5.  The CUDA-core stem forms the same products in another summation order; with one fp16
    plane that moves stored activations across fp16 rounding boundaries, and the flips propagate into a different
    rounding realisation of the whole network, as large as the mode's own error -- so it is held to the accuracy
    contract (within twice the TF32 arm's error against fp64) instead."""
    from hover_net_b200.models.hovernet.run_desc import infer_step
    sd = synth.make_state_dict(mode, nt, seed=0)
    net = _net(mode, nt, sd, "high")
    x = synth.make_patches(2, arch.PATCH_GEOMETRY[mode][0], seed=23)
    knobs = ("xform", "tc_prefetch", "stem_tc")
    default = {"stem_tc": 1, "xform": 1, "tc_prefetch": 4}
    try:
        ref = infer_step(x, net)
        assert np.isfinite(ref).all()
        for k in knobs:
            net.ctx.set_option(k, 0)
            out = infer_step(x, net)
            net.ctx.set_option(k, default[k])
            err = np.abs(out[..., -3:] - ref[..., -3:]).max()
            print("\n%s/%s high, %s=0: max diff %.3e" % (mode, nt, k, err))
            if k == "stem_tc":
                _assert_within_tf32_bar(out, x, sd, mode, nt, "%s/%s high stem_tc=0" % (mode, nt))
            else:
                assert err <= 3e-5, "%s=0 changes the output by %.3e" % (k, err)
        assert np.array_equal(infer_step(x, net), ref)
    finally:
        for k in knobs:
            net.ctx.set_option(k, default[k])   # tc_prefetch is process-wide
        net.ctx.close()


def test_high_referee_paths_run():
    """conv_path 1 (CUDA-core referee only) and 2 (per-layer self test) work on single-plane tensors; the self test
    reports the single product's error against fp32 arithmetic on the same stored operands.  The referee sums in
    another order, so its map is held to the accuracy contract (see test_high_kernel_variants_agree)."""
    from hover_net_b200.models.hovernet.run_desc import infer_step
    mode, nt = "fast", 6
    sd = synth.make_state_dict(mode, nt, seed=0)
    net = _net(mode, nt, sd, "high")
    x = synth.make_patches(1, 256, seed=9)
    ref = infer_step(x, net)
    net.ctx.set_option("conv_path", 1)
    r1 = infer_step(x, net)
    net.ctx.set_option("conv_path", 2)
    r2 = infer_step(x, net)
    log = net.ctx.debug_log()
    net.ctx.close()
    assert np.array_equal(r2, ref)
    _assert_within_tf32_bar(r1, x, sd, mode, nt, "high conv_path=1")
    lines = [l for l in log.splitlines() if "raw diff" in l]
    assert len(lines) > 50 and "CUDA ERROR" not in log


def _split_elements(mode, nt, B, H):
    """Elements of every activation buffer the plan stores as fp16 planes (cnn.cu Model::plan, default options)."""
    k = 5 if mode == "original" else 3
    nb = 3 if nt else 2
    s0 = H if mode == "fast" else H - 6
    n, si, ds = s0 * s0 * 64, s0, []
    for c1, c3, st in ((64, 256, 1), (128, 512, 2), (256, 1024, 2), (512, 2048, 2)):
        so = (si + st - 1) // st
        n += si * si * c1 + so * so * c1 + so * so * c3
        ds.append(so)
        si = so
    km1 = k - 1
    h3 = 2 * ds[3] - km1
    w8 = h3 - 8 * km1
    h2 = 2 * w8 - km1
    w4 = h2 - 4 * km1
    ho = 2 * w4
    n += (2 * ds[3]) ** 2 * 1024
    n += nb * (h3 * h3 * 512 + h2 * h2 * 256 + h3 * h3 * 128 + h2 * h2 * 128 + (2 * w8) ** 2 * 512 + ho * ho * 256)
    n += nb * ho * ho * 64
    return B * n


def test_high_plan_allocates_no_lo_planes():
    from hover_net_b200.models.hovernet.run_desc import infer_step
    mode, nt, B = "original", 5, 4
    sd = synth.make_state_dict(mode, nt, seed=0)
    x = synth.make_patches(B, 270, seed=1)
    got = {}
    for p in ("highest", "high"):
        net = _net(mode, nt, sd, p)
        infer_step(x, net)
        got[p] = net.ctx.counter("plan_bytes")
        net.ctx.close()
    lo_bytes = 2 * _split_elements(mode, nt, B, 270)
    print("\nplan_bytes highest %d, high %d, lo planes %d" % (got["highest"], got["high"], lo_bytes))
    assert got["high"] > 0 and got["highest"] - got["high"] >= lo_bytes
