"""Test-time augmentation (option "tta") on the H100: the device merge against a host merge of the plain forward on
host-made views (bit for bit), against an fp64 oracle TTA, the untouched default, errors, and every driver that goes
through the forward (tile, tile groups, validation, WSI)."""
import ctypes
import json
import os

import numpy as np
import pytest

from hover_net_b200 import arch, synth

import tta_ref

pytestmark = pytest.mark.gpu


def _net(mode, nt, sd=None, precision="highest", tta=False):
    from hover_net_b200.models.hovernet.net_desc import create_model
    net = create_model(mode=mode, input_ch=3, nr_types=nt, precision=precision, tta=tta)
    net.load_state_dict(sd if sd is not None else synth.make_state_dict(mode, nt, seed=0), strict=True)
    return net


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("precision", ["highest", "high"])
@pytest.mark.parametrize("mode,nt", [("original", None), ("original", 5), ("original", 6), ("fast", None),
                                     ("fast", 5), ("fast", 6)])
def test_merge_is_the_host_merge_of_the_plain_views(mode, nt, precision):
    """NP and HV of the TTA forward equal, bit for bit, the host merge (same inverse map, same fp32 sum order) of the
    plain forward's outputs on the eight host-made view batches; for batch tails and chunks that are not a multiple of
    8.  Rests on a patch's output not depending on the rest of its batch."""
    S = arch.PATCH_GEOMETRY[mode][0]
    x = synth.make_patches(33, S, seed=41)
    sd = synth.make_state_dict(mode, nt, seed=0)
    plain = _net(mode, nt, sd, precision)
    plain.ctx.set_option("chunk", 8)
    v = plain.ctx.forward(tta_ref.views(x))              # [8*33, h, w, C], slot 8i + t
    plain.ctx.close()
    v = v.reshape((33, 8) + v.shape[1:]).transpose(1, 0, 2, 3, 4)
    want = tta_ref.merge(v)
    net = _net(mode, nt, sd, precision, tta=True)
    try:
        for chunk in (32, 12):
            net.ctx.set_option("chunk", chunk)
            for B in (1, 3, 5, 33):
                got = net.ctx.forward(x[:B])
                assert got.shape == (B,) + want.shape[1:]
                assert np.array_equal(_bits(got[..., -3:]), _bits(want[:B, ..., -3:])), (chunk, B)
                if nt:
                    assert got[..., 0].min() >= 0 and got[..., 0].max() <= nt - 1
                    assert np.array_equal(got[..., 0], np.round(got[..., 0]))
    finally:
        net.ctx.close()


@pytest.mark.parametrize("mode,nt", [("original", None), ("original", 5), ("fast", 6)])
def test_tta_against_fp64_oracle(mode, nt):
    S = arch.PATCH_GEOMETRY[mode][0]
    x = synth.make_patches(2, S, seed=43)
    sd = synth.make_state_dict(mode, nt, seed=0)
    net = _net(mode, nt, sd, tta=True)
    out = net.ctx.forward(x)
    net.ctx.close()
    ref = tta_ref.oracle_tta(x, sd, mode, nt)
    hv_scale = max(1.0, float(np.abs(ref[..., -2:]).max()))
    e_np = float(np.abs(out[..., -3] - ref[..., -3]).max())
    e_hv = float(np.abs(out[..., -2:] - ref[..., -2:]).max()) / hv_scale
    print("\n%s/%s TTA vs fp64 oracle TTA: NP max %.3e, HV rel max %.3e" % (mode, nt, e_np, e_hv))
    assert e_np <= 1e-4 and e_hv <= 1e-4
    if nt:
        assert (out[..., 0] != ref[..., 0]).mean() < 2e-3


def test_default_and_switching():
    from hover_net_b200._lib import HvnError
    mode, nt = "original", 5
    sd = synth.make_state_dict(mode, nt, seed=0)
    x = synth.make_patches(3, 270, seed=45)
    fresh = _net(mode, nt, sd)
    a = fresh.ctx.forward(x)
    flops = fresh.ctx.counter("last_flops")
    assert fresh.ctx.counter("tta") == 0
    fresh.ctx.close()
    sw = _net(mode, nt, sd)
    try:
        sw.ctx.set_option("tta", 1)
        t = sw.ctx.forward(x)
        assert sw.ctx.counter("tta") == 1 and not np.array_equal(t, a)
        assert sw.ctx.counter("last_flops") == 8 * flops
        for bad in (2, -1):
            with pytest.raises(HvnError) as e:
                sw.ctx.set_option("tta", bad)
            assert e.value.code == -1
        sw.ctx.set_option("tta", 0)
        assert sw.ctx.counter("tta") == 0
        assert np.array_equal(_bits(sw.ctx.forward(x)), _bits(a)), "TTA off after a TTA run must be the plain forward"
        assert sw.ctx.counter("last_flops") == flops
    finally:
        sw.ctx.close()


def test_plan_bytes_count_the_tta_workspace():
    """The workspace (views and per-view probabilities) is per chunk, whatever the batch size."""
    mode, nt = "fast", 6
    net = _net(mode, nt, tta=True)
    try:
        net.ctx.set_option("chunk", 16)  # two inputs, 16 network patches per chunk
        x = synth.make_patches(4, 256, seed=47)
        net.ctx.forward(x[:2])
        two = net.ctx.counter("plan_bytes")
        net.ctx.forward(x)
        assert net.ctx.counter("plan_bytes") == two  # four inputs: the same plan twice
        net.ctx.set_option("tta", 0)
        net.ctx.forward(x)  # 4 patches: a quarter of the network buffers of the 16-patch plan
        plain4 = net.ctx.counter("plan_bytes")
        ws = 16 * (256 * 256 * 3 + 164 * 164 * (nt + 3) * 4)
        assert two == 4 * plain4 + ws, (two, plain4, ws)
    finally:
        net.ctx.close()


def test_rectangular_batch_is_invalid():
    from hover_net_b200._lib import HvnError
    net = _net("fast", 6, tta=True)
    try:
        x = np.zeros((1, 256, 264, 3), np.uint8)
        with pytest.raises(HvnError) as e:
            net.ctx.forward(x)
        assert e.value.code == -1 and "square" in str(e.value)
    finally:
        net.ctx.close()


def test_range_overflow_is_an_error_then_retry():
    """Stem activations pushed past 65504 under TTA: HVN_ERR_RANGE through the raw C ABI, then the binding's act_shift
    retry returns a finite map."""
    from hover_net_b200 import _lib
    from hover_net_b200.models.hovernet.run_desc import infer_step
    mode, nt = "fast", 6
    sd = dict(synth.make_state_dict(mode, nt, seed=0))
    sd["conv0./.weight"] = (sd["conv0./.weight"] * np.float32(3.0e5)).astype(np.float32)
    sd["conv0.bn.running_var"] = np.full_like(sd["conv0.bn.running_var"], 1.0)
    net = _net(mode, nt, sd, tta=True)
    x = synth.make_patches(1, 256, seed=3)
    out = np.empty((1, 164, 164, 4), np.float32)
    L = _lib.lib()
    rc = L.hvn_forward(net.ctx._h, x.ctypes.data_as(ctypes.c_void_p), 1, 256, 256, out.ctypes.data_as(ctypes.c_void_p))
    assert rc == -6 and b"act_shift" in L.hvn_last_error()
    out = infer_step(x, net)
    assert np.isfinite(out).all() and net.ctx.counter("act_shift") > 0 and net.ctx.counter("tta") == 1
    net.ctx.close()


def _manager(mode, nt, batch):
    from hover_net_b200.infer.tile import InferManager
    mgr = InferManager(method={"model_args": {"nr_types": nt, "mode": mode, "tta": True},
                               "model_path": synth.make_state_dict(mode, nt, seed=0)}, type_info_path=None)
    mgr.patch_input_shape, mgr.patch_output_shape = {"fast": (256, 164), "original": (270, 80)}[mode]
    mgr.batch_size = batch
    return mgr


def _img(h, w, seed):
    k = -(-max(h, w) // 256)
    tiles = synth.make_patches(k * k, 256, seed=seed)
    big = np.concatenate([np.concatenate(list(tiles[r * k:(r + 1) * k]), 1) for r in range(k)], 0)
    return np.ascontiguousarray(big[:h, :w])


def _same_instances(ia, da, ib, db):
    assert np.array_equal(ia, ib)
    assert list(da.keys()) == list(db.keys())
    for k in da:
        x, y = da[k], db[k]
        assert np.array_equal(x["bbox"], y["bbox"]) and np.array_equal(x["centroid"], y["centroid"])
        assert np.array_equal(x["contour"], y["contour"])
        assert x["type"] == y["type"] and x["type_prob"] == y["type_prob"]


@pytest.mark.parametrize("mode,nt", [("fast", 6), ("original", 5)])
def test_tile_mode(mode, nt):
    from hover_net_b200.infer import tile
    from hover_net_b200.models.hovernet.post_proc import process
    from hover_net_b200.models.hovernet.run_desc import infer_step
    mgr = _manager(mode, nt, batch=5)
    win, msk = mgr.patch_input_shape, mgr.patch_output_shape
    try:
        assert mgr.net.ctx.counter("tta") == 1
        img = _img(300, 420, 51)
        pred, inst, info = mgr.infer_image(img)
        padded, pinfo, _ = tile._prepare_patching(img, win, msk, True)
        outs = infer_step(np.stack([padded[y:y + win, x:x + win] for y, x, _, _ in pinfo]), mgr.net)
        ref_map = tile._stitch(list(pinfo), list(outs), img.shape)
        assert np.array_equal(_bits(pred), _bits(ref_map))
        ri, rinfo = process(ref_map, nr_types=nt, return_centroids=True)
        if mode == "fast":  # the synthetic original-mode checkpoint yields no nuclei (DESIGN §6)
            assert len(rinfo) > 0
        _same_instances(inst, info, ri, rinfo)
        imgs = [_img(h, w, 52 + i) for i, (h, w) in enumerate([(256, 256), (300, 420), (100, 80)])]
        singles = [mgr.infer_image(im) for im in imgs]
        group = mgr.infer_images(imgs)  # batches of 5 patches straddle images
        for (pg, ig, dg), (ps, is_, ds) in zip(group, singles):
            assert np.array_equal(_bits(pg), _bits(ps))
            _same_instances(ig, dg, is_, ds)
    finally:
        mgr.net.ctx.close()


def test_validation_counts():
    """hvn_valid under TTA gives the counts of the reference's proc_valid_step_output over valid_step, same model."""
    from hover_net_b200.models.hovernet import run_desc
    from hover_net_b200.models.hovernet.targets import cropping_center
    from oracle import targets_oracle as TO
    mode, nt = "original", 5
    net = _net(mode, nt, tta=True)
    try:
        size = arch.PATCH_GEOMETRY[mode][0]
        imgs = synth.make_patches(3, size, seed=53)
        inst = np.stack([synth.synth_instances(size, size, seed=530 + i) for i in range(3)])
        typ = np.where(inst > 0, inst % nt, 0).astype(np.int32)
        counts, sse, flags = net.ctx.valid(imgs, inst, typ)
        assert not flags.any()
        h, w = net.ctx.out_shape(size, size)[:2]
        true_hv = np.stack([cropping_center(TO.hv_map(m, (h, w))[0], (h, w)) for m in inst])
        inst_c = cropping_center(inst, (h, w), batch=True)
        typ_c = cropping_center(typ, (h, w), batch=True)
        batch = {"img": imgs, "np_map": (inst_c > 0).astype(np.int64), "hv_map": true_hv, "tp_map": typ_c}
        raw = run_desc.valid_step(batch, ({"net": {"desc": net}}, None))["raw"]
        mirror = run_desc.proc_valid_step_output(raw, nr_types=nt)["scalar"]
        tc = [(counts[3 + 2 * k], counts[4 + 2 * k]) for k in range(nt)]
        got = run_desc.valid_scalars(counts[0], counts[1], counts[2], tc, sse, inst_c.size)
        assert list(got) == list(mirror)
        for k in got:
            if k == "hv_mse":
                assert abs(float(got[k]) - float(mirror[k])) <= 1e-5 * abs(float(mirror[k]))
            else:
                assert got[k] == mirror[k], k
    finally:
        net.ctx.close()


def test_cli_wsi_with_tta(tmp_path):
    """`run_infer.py --tta ... wsi` on the synthetic slide of the WSI driver test completes, on a TTA context."""
    import cv2
    from hover_net_b200 import run_infer
    from hover_net_b200.infer import wsi
    h, w = 600, 700
    base = synth.make_patches(12, 256, seed=60)
    img = np.concatenate([np.concatenate(list(base[r * 3:(r + 1) * 3]), 1) for r in range(3)], 0)[:h, :w].copy()
    os.makedirs(tmp_path / "in")
    np.save(str(tmp_path / "in" / "slide.npy"), img)
    np.savez(str(tmp_path / "ckpt.npz"), **synth.make_state_dict("fast", 6, seed=0))
    os.makedirs(tmp_path / "msk")
    cv2.imwrite(str(tmp_path / "msk" / "slide.png"), np.full((h // 8, w // 8), 255, np.uint8))
    argv = ["--nr_types=6", "--model_mode=fast", "--model_path=%s" % (tmp_path / "ckpt.npz"), "--batch_size=8", "--tta",
            "wsi", "--input_dir=%s" % (tmp_path / "in"), "--output_dir=%s" % (tmp_path / "out"),
            "--cache_path=%s" % (tmp_path / "cache"), "--input_mask_dir=%s" % (tmp_path / "msk"), "--chunk_shape=500",
            "--tile_shape=256", "--ambiguous_size=32"]
    cmd, margs, rargs, _ = run_infer.parse(argv)
    assert cmd == "wsi" and margs["method"]["model_args"]["tta"] is True
    margs["method"]["model_args"]["device"] = 0
    mgr = wsi.InferManager(**margs)
    try:
        mgr.process_wsi_list(rargs)
        assert mgr.net.ctx.counter("tta") == 1
        js = json.load(open(str(tmp_path / "out" / "slide.json")))
        assert js["mag"] == 40 and len(js["nuc"]) > 0
    finally:
        mgr.net.ctx.close()
