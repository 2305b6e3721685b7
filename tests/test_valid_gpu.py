"""GPU checks of the training targets (hvn_targets*) and the fused validation step (hvn_valid*): the device HV
maps equal the reference's goldens and the numpy oracle bit for bit, and the validation counts equal the host
mirror of proc_valid_step_output applied to the engine's own forward maps plus oracle targets."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from hover_net_b200 import arch, synth
from oracle import targets_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def ctx():
    from hover_net_b200.models.hovernet.post_proc import _ctx
    return _ctx()


def _same_as_oracle(ctx, maps, crop):
    hv, flags = ctx.targets(maps, crop)
    for m in range(maps.shape[0]):
        ohv, of = O.hv_map(maps[m], crop)
        assert flags[m] == of, m
        if of == 0:
            assert hv[m].tobytes() == ohv.tobytes(), m
    return hv, flags


def test_hv_maps_match_reference():
    from hover_net_b200.models.hovernet import targets as T
    g = np.load(os.path.join(GOLDEN, "targets_cases.npz"))
    res = json.loads(str(g["results"]))
    for k, rec in enumerate(res):
        ann, crop = g["ann_%d" % k], [int(v) for v in g["crop_%d" % k]]
        if "raises" in rec:
            with pytest.raises(ValueError):
                T.gen_instance_hv_map(ann, crop)
            with pytest.raises(ValueError):
                T.gen_targets(ann, crop)
            continue
        hv = T.gen_instance_hv_map(ann, crop)
        assert hv.tobytes() == g["hv_%d" % k].tobytes(), rec["name"]
        tg = T.gen_targets(ann, crop)
        assert np.array_equal(tg["hv_map"], g["tgt_hv_%d" % k]) and np.array_equal(tg["np_map"], g["tgt_np_%d" % k])


def test_flags_match_oracle_on_goldens(ctx):
    g = np.load(os.path.join(GOLDEN, "targets_cases.npz"))
    for k in range(len(json.loads(str(g["results"])))):
        ann = g["ann_%d" % k]
        _same_as_oracle(ctx, ann[None], tuple(int(v) for v in g["crop_%d" % k]))


def test_batched_540_and_single(ctx):
    maps = np.stack([synth.synth_instances(540, 540, seed=40 + i, density=1.0 / 500.0) for i in range(6)])
    maps[1] = np.where(maps[1] > 0, (maps[1] + 2) // 3, 0)  # ids in several pieces
    assert all(len(np.unique(m)) > 300 for m in maps[2:])
    hv, flags = _same_as_oracle(ctx, maps, (164, 164))
    assert not flags.any() and np.abs(hv).max() == 1.0
    for m in range(maps.shape[0]):
        h1, f1 = ctx.targets(maps[m], (164, 164))
        assert f1[0] == flags[m] and h1[0].tobytes() == hv[m].tobytes()


def test_random_ids_all_small(ctx):
    rng = np.random.default_rng(5)
    maps = rng.integers(0, 2 ** 20, (3, 270, 270)).astype(np.int32)
    maps[:2, 0, 0] = 0
    maps[2][maps[2] == 0] = 7  # no background pixel: the reference rejects this map
    hv, flags = _same_as_oracle(ctx, maps, (80, 80))
    assert not hv.any() and list(flags) == [0, 0, 1]


def test_ids_near_int32_max(ctx):
    from hover_net_b200._lib import HvnError
    base = synth.synth_instances(270, 270, seed=9)
    n = int(base.max())
    m = np.where(base > 0, base + (2 ** 31 - 1 - n - 10 - n), 0).astype(np.int32)  # room for every component
    _same_as_oracle(ctx, m[None], (80, 80))
    top = np.where(base > 0, base + (2 ** 31 - 1 - n), 0).astype(np.int32)  # largest id 2^31 - 1
    with pytest.raises(ValueError):
        O.hv_map(top, (80, 80))
    with pytest.raises(HvnError) as e:
        ctx.targets(top, (80, 80))
    assert e.value.code == -1 and "2^31" in str(e.value)


def test_negative_id_is_invalid(ctx):
    from hover_net_b200._lib import HvnError
    a = synth.synth_instances(270, 270, seed=3)
    a[100, 100] = -5
    with pytest.raises(HvnError) as e:
        ctx.targets(a, (80, 80))
    assert e.value.code == -1 and "negative" in str(e.value)
    with pytest.raises(HvnError) as e:
        ctx.targets(a[:50, :50] * 0, (51, 51))
    assert e.value.code == -1


# ------------------------------------------------------------------------------------------------ validation
def _net(mode, nt, precision="highest"):
    from hover_net_b200.models.hovernet.net_desc import create_model
    net = create_model(mode=mode, input_ch=3, nr_types=nt, precision=precision)
    net.load_state_dict(synth.make_state_dict(mode, nt, seed=0), strict=True)
    return net


def _batch(mode, nt, B, seed):
    size = arch.PATCH_GEOMETRY[mode][0]
    imgs = synth.make_patches(B, size, seed=seed)
    inst = np.stack([synth.synth_instances(size, size, seed=seed * 10 + i) for i in range(B)])
    typ = np.where(inst > 0, inst % max(nt or 1, 1), 0).astype(np.int32) if nt else None
    return imgs, inst, typ


def _host_counts(prob, tp, hv_pred, inst_c, typ_c, hv_true, nt):
    pn, tn = prob > np.float32(0.5), inst_c > 0
    c = [int((pn == tn).sum()), int((pn & tn).sum()), int(pn.sum() + tn.sum())]
    for k in range(nt or 0):
        pk, tk = tp == k, typ_c == k
        c += [int((pk & tk).sum()), int(pk.sum() + tk.sum())]
    d = (hv_pred - hv_true).astype(np.float32)
    return np.array(c, np.int64), float((d.astype(np.float64) ** 2).sum())


@pytest.mark.parametrize("mode,nt,precision", [("original", None, "highest"), ("original", 5, "highest"),
                                               ("fast", 6, "highest"), ("original", 5, "high")])
def test_valid_counts_equal_host_mirror(mode, nt, precision):
    from hover_net_b200.models.hovernet import run_desc
    from hover_net_b200.models.hovernet.targets import cropping_center
    net = _net(mode, nt, precision)
    ctx = net.ctx
    imgs, inst, typ = _batch(mode, nt, 3, seed=21)
    counts, sse, flags = ctx.valid(imgs, inst, typ)
    assert not flags.any()
    pred = ctx.forward(imgs)
    h, w = pred.shape[1:3]
    true_hv = np.stack([cropping_center(O.hv_map(m, (h, w))[0], (h, w)) for m in inst])
    inst_c = cropping_center(inst, (h, w), batch=True)
    typ_c = cropping_center(typ, (h, w), batch=True) if nt else None
    want, want_sse = _host_counts(pred[..., -3], pred[..., 0] if nt else None, pred[..., -2:], inst_c, typ_c,
                                  true_hv, nt)
    assert np.array_equal(counts, want), (counts, want)
    assert abs(sse - want_sse) <= 1e-9 * want_sse
    raw = {"imgs": imgs, "true_np": (inst_c > 0).astype(np.int64), "true_hv": true_hv,
           "prob_np": np.ascontiguousarray(pred[..., -3]), "pred_hv": np.ascontiguousarray(pred[..., -2:])}
    if nt:
        raw["true_tp"], raw["pred_tp"] = typ_c.astype(np.int64), np.ascontiguousarray(pred[..., 0])
    mirror = run_desc.proc_valid_step_output(raw, nr_types=nt)["scalar"]
    tc = [(counts[3 + 2 * k], counts[4 + 2 * k]) for k in range(nt)] if nt else None
    got = run_desc.valid_scalars(counts[0], counts[1], counts[2], tc, sse, inst_c.size)
    assert list(got) == list(mirror)
    for k in got:
        if k == "hv_mse":
            assert abs(float(got[k]) - float(mirror[k])) <= 1e-5 * abs(float(mirror[k]))
        else:
            assert got[k] == mirror[k], k
    # device pointers, same batch
    B, H, W = inst.shape
    nc = counts.size
    d = [ctx.malloc(n) for n in (imgs.nbytes, inst.nbytes, inst.nbytes, nc * 8, 8, B * 4)]
    try:
        ctx.h2d(d[0], imgs, imgs.nbytes)
        ctx.h2d(d[1], inst, inst.nbytes)
        if nt:
            ctx.h2d(d[2], np.ascontiguousarray(typ), typ.nbytes)
        ctx.valid_dev(d[0], d[1], d[2] if nt else None, B, H, W, d[3], d[4], d[5])
        c2, s2 = np.zeros(nc, np.int64), np.zeros(1, np.float64)
        ctx.d2h(c2, d[3], nc * 8)
        ctx.d2h(s2, d[4], 8)
        assert np.array_equal(c2, counts) and abs(s2[0] - sse) <= 1e-12 * sse
    finally:
        for p in d:
            ctx.free(p)


def test_valid_against_torch_oracle():
    """Counts from the torch oracle's fp32 forward (TF32 off): they may differ only at pixels whose probability lies
    within 1e-4 of the 0.5 threshold."""
    import torch
    from oracle import hovernet_torch as TO
    mode, nt = "original", 5
    net = _net(mode, nt)
    imgs, inst, typ = _batch(mode, nt, 2, seed=22)
    counts, _, _ = net.ctx.valid(imgs, inst, typ)
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ref = TO.infer_step(imgs, TO.to_torch_state_dict(synth.make_state_dict(mode, nt, seed=0)), mode, nt,
                            dtype=torch.float32, device="cuda")
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    h, w = ref.shape[1:3]
    from hover_net_b200.models.hovernet.targets import cropping_center
    inst_c = cropping_center(inst, (h, w), batch=True)
    pn, tn = ref[..., -3] > np.float32(0.5), inst_c > 0
    near = int((np.abs(ref[..., -3].astype(np.float64) - 0.5) <= 1e-4).sum())
    assert abs(int(counts[0]) - int((pn == tn).sum())) <= near
    assert abs(int(counts[1]) - int((pn & tn).sum())) <= near
    assert abs(int(counts[2]) - int(pn.sum() + tn.sum())) <= near


def test_valid_rejects_bad_input():
    from hover_net_b200._lib import HvnError
    net = _net("original", 5)
    imgs, inst, typ = _batch("original", 5, 1, seed=23)
    with pytest.raises(HvnError):
        net.ctx.valid(imgs, inst, None)  # a typed model needs the type map
    bad = inst.copy()
    bad[0, 0, 0] = -1
    with pytest.raises(HvnError) as e:
        net.ctx.valid(imgs, bad, typ)
    assert e.value.code == -1
    full = np.ones_like(inst)
    _, _, flags = net.ctx.valid(imgs, full, typ)
    assert flags[0] & 1


def test_run_valid_end_to_end(tmp_path):
    from hover_net_b200.dataloader.train_loader import FileLoader
    from hover_net_b200.models.hovernet import run_desc, targets
    from test_oracle_targets import _write_patches
    mode, nt = "original", 5
    paths = _write_patches(tmp_path, 5, 300, True, seed=3)
    ck = tmp_path / "ck.npz"
    np.savez(ck, **{k: np.asarray(v) for k, v in synth.make_state_dict(mode, nt, seed=0).items()})
    out = tmp_path / "scal.json"
    r = subprocess.run([sys.executable, "-m", "hover_net_b200.run_valid", "--model_path", str(ck), "--valid_dir",
                        str(tmp_path), "--nr_types", str(nt), "--batch_size", "2", "--json", str(out)],
                       cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    printed = dict(line.split(": ") for line in r.stdout.strip().split("\n"))
    got = json.loads(out.read_text())
    assert list(got) == ["np_acc", "np_dice"] + ["tp_dice_%d" % k for k in range(nt)] + ["hv_mse"]
    assert {k: float(v) for k, v in printed.items()} == got
    # the reference protocol on the host: FileLoader + valid_step + proc_valid_step_output over all patches
    net = _net(mode, nt)
    fl = FileLoader(paths, with_type=True, input_shape=[270, 270], mask_shape=[80, 80], mode="valid",
                    target_gen=(targets.gen_targets, {}))
    items = [fl[i] for i in range(len(fl))]
    batch = {k: np.stack([it[k] for it in items]) for k in items[0]}
    raw = run_desc.valid_step(batch, ({"net": {"desc": net}}, {}))["raw"]
    want = run_desc.proc_valid_step_output(raw, nr_types=nt)["scalar"]
    for k, v in want.items():
        if k == "hv_mse":
            assert abs(got[k] - float(v)) <= 1e-5 * abs(float(v))
        else:
            assert got[k] == float(v), k
