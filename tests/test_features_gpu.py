"""hvn_inst_features(_dev) against the float64 restatement (tests/features_ref.py): columns 0-16 bit for bit
(orientation within 4 ulp), np_prob_mean to a relative 1e-12; and the feature outputs of process, tile mode and WSI
mode against the restatement on the nuclei they describe."""
import json
import os

import numpy as np
import pytest

import features_ref as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from hover_net_b200 import _lib
    c = _lib.Context(0)
    yield c
    c.close()


def _ulps(a, b):
    return np.abs(a.view(np.int64) - b.view(np.int64))


def assert_features(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    exact = [k for k in range(17) if k != 9]
    g, w = got[:, exact], want[:, exact]
    same = (g.view(np.int64) == w.view(np.int64)) | (np.isnan(g) & np.isnan(w))
    assert same.all(), "columns differ at %s: %s vs %s" % (np.argwhere(~same)[:5], g[~same][:5], w[~same][:5])
    o_g, o_w = got[:, 9], want[:, 9]
    assert (_ulps(o_g, o_w) <= 4).all(), (o_g, o_w)
    n_g, n_w = got[:, 17], want[:, 17]
    assert np.array_equal(np.isnan(n_g), np.isnan(n_w))
    ok = ~np.isnan(n_w)
    assert (np.abs(n_g[ok] - n_w[ok]) <= 1e-12 * np.abs(n_w[ok])).all()


def _inputs(inst, seed, channels=4):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, inst.shape + (3,), dtype=np.uint8)
    pred = rng.uniform(0, 1, inst.shape + (channels,)).astype(np.float32)
    return img, pred


CASES = F.edge_maps() + [("seeded%d" % s, F.seeded_map(160, 200, s, n=60)) for s in range(2)]


@pytest.mark.parametrize("name,inst", CASES, ids=[n for n, _ in CASES])
@pytest.mark.parametrize("with_img,with_pred", [(True, True), (False, False), (True, False), (False, True)])
def test_maps_match_restatement(ctx, name, inst, with_img, with_pred):
    table = F.table_of(inst)
    pts, offs = F.cv2_contours(inst, table)
    img, pred = _inputs(inst, 5, 3 if name.startswith("seeded1") else 4)
    img, pred = (img if with_img else None), (pred if with_pred else None)
    got = ctx.inst_features(inst, table, pts, offs, image=img, pred=pred)
    assert_features(got, F.features(inst, table, pts, offs, img, pred))


def test_u8_extremes(ctx):
    inst = F.seeded_map(64, 64, 3, n=12)
    table = F.table_of(inst)
    pts, offs = F.cv2_contours(inst, table)
    for v in (0, 255):
        img = np.full(inst.shape + (3,), v, np.uint8)
        got = ctx.inst_features(inst, table, pts, offs, image=img)
        assert_features(got, F.features(inst, table, pts, offs, img))
        assert (got[:, 14:17] == 0).all() and (got[:, 11:14] == v).all()


@pytest.mark.parametrize("n", [1, 2, 3, 511, 512, 513, 2000])
def test_point_sets_on_both_sides_of_the_shared_cap(ctx, n):
    """The contour pass on arbitrary point lists (with repeats and collinear runs) of n points: rows up to 512 points
    are hulled in shared memory, longer ones in global scratch.  Two rows, so the scratch offsets are exercised."""
    rng = np.random.default_rng(n)
    inst = np.zeros((90, 120), np.int32)
    inst[5:80, 10:110] = 1
    inst[82:90, 0:120] = 2
    table = F.table_of(inst)
    p1 = np.stack([rng.integers(10, 110, n), rng.integers(5, 80, n)], 1)
    p1[: n // 4] = p1[0]                                    # repeats
    p2 = np.stack([rng.integers(0, 120, n + 7), np.full(n + 7, 85)], 1)  # collinear
    pts = np.concatenate([p1, p2]).astype(np.int32)
    offs = np.array([0, n, 2 * n + 7], np.int32)
    img, pred = _inputs(inst, n)
    got = ctx.inst_features(inst, table, pts, offs, image=img, pred=pred)
    assert_features(got, F.features(inst, table, pts, offs, img, pred))
    assert got[1, 3] == 0.0  # collinear: convex_area 0


def test_zero_rows(ctx):
    inst = np.zeros((8, 8), np.int32)
    got = ctx.inst_features(inst, np.zeros((0, 10), np.int64), np.zeros((0, 2), np.int32), np.zeros(1, np.int32))
    assert got.shape == (0, 18)


def _packed(maps, seed):
    tables, ptsl, offs, ro, imgs, preds = [], [], [0], [0], [], []
    for m in maps:
        t = F.table_of(m)
        p, o = F.cv2_contours(m, t)
        tables.append(t)
        ptsl.append(p)
        offs.extend((o[1:] + offs[-1]).tolist())
        ro.append(ro[-1] + len(t))
        img, pred = _inputs(m, seed + len(imgs))
        imgs.append(img)
        preds.append(pred)
    return (np.concatenate(tables), np.concatenate(ptsl), np.array(offs, np.int32), np.array(ro, np.int32), imgs,
            preds)


def _dev_call(ctx, maps, table, pts, offs, ro, imgs, preds):
    """hvn_inst_features_dev on device copies of the packed inputs; returns feats."""
    cat = lambda arrs: np.ascontiguousarray(np.concatenate([a.reshape(-1) for a in arrs]))  # noqa: E731
    host = [cat(maps).astype(np.int32), cat(imgs), cat(preds), np.ascontiguousarray(table), np.ascontiguousarray(ro),
            np.ascontiguousarray(pts), np.ascontiguousarray(offs)]
    d = [ctx.malloc(max(1, a.nbytes)) for a in host]
    n = len(table)
    d_f = ctx.malloc(max(1, n * 18 * 8))
    try:
        for dp, a in zip(d, host):
            ctx.h2d(dp, a, a.nbytes)
        shapes = np.array([m.shape for m in maps], np.int32)
        outs = []
        for _ in range(2):
            ctx.inst_features_dev(len(maps), shapes, d[0], d[1], d[2], 4, d[3], d[4], n, d[5], d[6], d_f)
            f = np.empty((n, 18), np.float64)
            ctx.d2h(f, d_f, f.nbytes)
            ctx.sync()
            outs.append(f)
        return outs
    finally:
        for dp in d + [d_f]:
            ctx.free(dp)


def test_packed_group_dev_host_and_determinism(ctx):
    maps = [m for _, m in CASES]
    table, pts, offs, ro, imgs, preds = _packed(maps, 40)
    host = ctx.inst_features(maps, table, pts, offs, row_offs=ro, image=imgs, pred=preds)
    d1, d2 = _dev_call(ctx, maps, table, pts, offs, ro, imgs, preds)
    assert np.array_equal(d1.view(np.int64), d2.view(np.int64))      # repeated calls are bit-identical
    assert np.array_equal(host.view(np.int64), d1.view(np.int64))    # the host twin is the _dev call
    for k, m in enumerate(maps):
        r0, r1 = int(ro[k]), int(ro[k + 1])
        want = F.features(m, table[r0:r1], pts, offs[r0:r1 + 1], imgs[k], preds[k])
        assert_features(host[r0:r1], want)


def test_profile_stage_and_launch_count(ctx):
    inst = F.seeded_map(64, 64, 1, n=10)
    table = F.table_of(inst)
    pts, offs = F.cv2_contours(inst, table)
    before = ctx.counter("pp_launches")
    ctx.set_option("profile", 1)
    try:
        ctx.inst_features(inst, table, pts, offs)
        assert ctx.stage_ms("features") > 0
    finally:
        ctx.set_option("profile", 0)
    assert ctx.counter("pp_launches") == before + 2


def test_errors(ctx):
    from hover_net_b200 import _lib
    inst = F.seeded_map(40, 40, 2, n=5)
    table = F.table_of(inst)
    pts, offs = F.cv2_contours(inst, table)
    pred = np.zeros((40, 40, 2), np.float32)
    n = len(table)
    L, h = _lib.lib(), ctx._h
    sh = np.array([[40, 40]], np.int32)
    feats = np.empty((n, 18))

    def call(shapes=sh, pred_=None, C=0, tab=table, ro=np.array([0, n], np.int32), n_rows=n, p=pts, po=offs):
        return L.hvn_inst_features(h, len(shapes), _lib._ptr(shapes), _lib._ptr(inst), None, _lib._ptr(pred_), C,
                                   _lib._ptr(np.ascontiguousarray(tab)), _lib._ptr(ro), n_rows, _lib._ptr(p),
                                   _lib._ptr(np.ascontiguousarray(po, dtype=np.int32)), _lib._ptr(feats))
    assert call() == 0
    assert call(pred_=pred, C=2) == -1                                    # C < 3 with a prediction map
    assert call(shapes=np.array([[0, 40]], np.int32)) == -1               # bad shape
    assert call(ro=np.array([0, n - 1], np.int32)) == -1                  # row_offs[n_maps] != n_rows
    assert call(ro=np.array([1, n], np.int32)) == -1                      # row_offs[0] != 0
    bad = table.copy()
    bad[0, 3] = 41                                                        # bbox outside the map
    assert call(tab=bad) == -1
    bad = table.copy()
    bad[0, 3] = bad[0, 1]                                                 # empty bbox
    assert call(tab=bad) == -1
    po = offs.copy()
    po[1], po[2] = po[2], po[1]                                           # falling point offsets
    assert call(po=po) == -1
    p = pts.copy()
    p[0] = [int(table[0, 4]), int(table[0, 1])]                           # a point outside its row's bbox
    assert call(p=p) == -1
    # interior offsets outside the call's point range [pt_offs[0], pt_offs[n_rows]], the neighbouring row's own pair in
    # order: the check reads no point of that row
    for v in (-10 ** 8, 10 ** 9):
        po = offs.copy()
        po[1] = v
        assert call(po=po) == -1
        with pytest.raises(_lib.HvnError):
            ctx.inst_features(inst, table, pts, po)
    # pt_offs[n_rows] is the point count the C call is told; the Python wrapper holds it to the array it is given
    po = offs.copy()
    po[n] = 10 ** 9
    with pytest.raises(ValueError):
        ctx.inst_features(inst, table, pts, po)
    assert call() == 0                                                    # the context is still usable


def test_non_uint8_image_is_an_error(ctx):
    inst = F.seeded_map(40, 40, 2, n=5)
    table = F.table_of(inst)
    pts, offs = F.cv2_contours(inst, table)
    for dt in (np.float32, np.uint16):
        with pytest.raises(ValueError):
            ctx.inst_features(inst, table, pts, offs, image=np.zeros((40, 40, 3), dt))


# ---- end to end --------------------------------------------------------------------------------------------------
def _check_records(info, inst, img, pred):
    """Every record's "features" equals the restatement on its nucleus: the pixels of its id in `inst` within its
    box, its contour, `img` and the NP channel of `pred`.  The box is the contour's (an outer border reaches every
    extreme row and column of its nucleus): the reference's WSI merge shifts "bbox" by the tile corner in (x, y) order,
    so a slide-level bbox is off wherever a tile's row and column offsets differ."""
    from hover_net_b200 import _lib
    np_map = None if pred is None else pred[..., pred.shape[-1] - 3]
    assert len(info) > 0
    for iid, v in info.items():
        c = np.asarray(v["contour"]).reshape(-1, 2)
        cmin, rmin = c.min(0).tolist()
        cmax, rmax = (c.max(0) + 1).tolist()
        want = F.row_features(inst, [int(iid), rmin, cmin, rmax, cmax], np.asarray(v["contour"]), img, np_map)
        got = np.array([v["features"].get(k, np.nan) for k in _lib.FEATURE_NAMES])
        assert_features(got[None], want[None])


def test_process_features():
    from hover_net_b200 import synth
    from hover_net_b200.models.hovernet import post_proc
    pm = synth.synth_pred_map(200, 240, 6, 3)
    img = np.random.default_rng(4).integers(0, 256, (200, 240, 3), dtype=np.uint8)
    inst0, info0 = post_proc.process(pm, nr_types=6, return_centroids=True)
    inst, info = post_proc.process_features(pm, nr_types=6, image=img)
    assert np.array_equal(inst, inst0) and list(info) == list(info0)
    for k in info:
        assert {kk: vv for kk, vv in info[k].items() if kk != "features"}.keys() == info0[k].keys()
        assert np.array_equal(info[k]["contour"], info0[k]["contour"])
    _check_records(info, inst, img, pm)
    _, info_n = post_proc.process_features(pm, nr_types=6)  # no image: the colour columns are left out
    assert all("mean_r" not in v["features"] and "np_prob_mean" in v["features"] for v in info_n.values())


def _tile_img(h, w, seed):
    from hover_net_b200 import synth
    k = -(-max(h, w) // 256)
    tiles = synth.make_patches(k * k, 256, seed=seed)
    big = np.concatenate([np.concatenate(list(tiles[r * k:(r + 1) * k]), 1) for r in range(k)], 0)
    return np.ascontiguousarray(big[:h, :w])


@pytest.fixture(scope="module")
def net():
    from hover_net_b200 import synth
    from hover_net_b200.models.hovernet.net_desc import create_model
    n = create_model(mode="fast", input_ch=3, nr_types=6)
    n.load_state_dict(synth.make_state_dict("fast", 6, seed=0), strict=True)
    yield n
    n.ctx.close()


def test_tile_group_features(net):
    """A mixed-size group straight from hvn_infer_tiles: the synchronous call and the enqueued TilesJob."""
    c = net.ctx
    imgs = [_tile_img(256, 256, 1), _tile_img(300, 420, 2), _tile_img(100, 80, 3), _tile_img(256, 256, 4)]
    plain = c.infer_tiles(imgs, 256, 8)
    res = c.infer_tiles(imgs, 256, 8, features=True)
    job = c.infer_tiles_begin(imgs, 256, 8, want_pred=False, features=True).result()
    assert sum(len(r[2]) for r in res) > 0
    for img, a, b, p in zip(imgs, res, job, plain):
        pred, inst, table, offs, pts, feats = a
        assert np.array_equal(inst, p[1]) and np.array_equal(table, p[2]) and np.array_equal(pts, p[4])
        assert b[0] is None and np.array_equal(b[5].view(np.int64), feats.view(np.int64))
        assert_features(feats, F.features(inst, table, pts, offs, img, pred))
    # a group rerun after capacity failures (table, then points) measures the same rows
    small = c.infer_tiles(imgs, 256, 8, features=True, rows_cap=1, pts_cap=1)
    for a, b in zip(res, small):
        assert all(np.array_equal(x, y) for x, y in zip(a[1:5], b[1:5]))
        assert np.array_equal(a[5].view(np.int64), b[5].view(np.int64))


def test_tile_group_features_range_retry():
    """A checkpoint whose activations leave the fp16 range (as in test_tile_group_gpu.py::test_range_retry_in_group):
    the group with features raises act_shift and reruns on the device, and then equals the group without features at
    that act_shift; its features equal the restatement."""
    from hover_net_b200 import synth
    from hover_net_b200.models.hovernet.net_desc import create_model
    sd = dict(synth.make_state_dict("fast", 6, seed=0))
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
    sd["conv0./.weight"] = (sd["conv0./.weight"] * np.float32(3.0e5)).astype(np.float32)
    imgs = [synth.make_patches(1, 256, seed=33)[0], _tile_img(300, 420, 32)]
    n = create_model(mode="fast", input_ch=3, nr_types=6)
    n.load_state_dict(sd, strict=True)
    try:
        c = n.ctx
        assert c.counter("act_shift") == 0
        res = c.infer_tiles(imgs, 256, 8, features=True)
        assert c.counter("act_shift") > 0
        plain = c.infer_tiles(imgs, 256, 8)
        for img, a, p in zip(imgs, res, plain):
            assert all(np.array_equal(x, y) for x, y in zip(a[:5], p[:5]))
            assert_features(a[5], F.features(a[1], a[2], a[4], a[3], img, a[0]))
    finally:
        n.ctx.close()


def test_tile_mode_save_features(tmp_path):
    import cv2
    import scipy.io as sio
    from hover_net_b200 import _lib, synth
    from hover_net_b200.infer.tile import InferManager
    os.makedirs(tmp_path / "in")
    imgs = {"a": _tile_img(300, 420, 7), "b": _tile_img(200, 180, 8), "c": _tile_img(300, 420, 9)}
    for k, im in imgs.items():
        cv2.imwrite(str(tmp_path / "in" / ("%s.png" % k)), cv2.cvtColor(im, cv2.COLOR_RGB2BGR))
    mgr = InferManager(method={"model_args": {"nr_types": 6, "mode": "fast"},
                               "model_path": synth.make_state_dict("fast", 6, seed=0)}, type_info_path=None)
    run = {"batch_size": 8, "patch_input_shape": 256, "patch_output_shape": 164, "input_dir": str(tmp_path / "in"),
           "mem_usage": 0.1}
    mgr.process_file_list(dict(run, output_dir=str(tmp_path / "raw"), save_raw_map=True, save_features=True))
    mgr.process_file_list(dict(run, output_dir=str(tmp_path / "plain"), save_features=True))
    mgr.process_file_list(dict(run, output_dir=str(tmp_path / "off")))
    for k, im in imgs.items():
        mat = sio.loadmat(str(tmp_path / "raw" / "mat" / ("%s.mat" % k)))
        js = json.load(open(str(tmp_path / "raw" / "json" / ("%s.json" % k))))["nuc"]
        info = {int(i): v for i, v in js.items()}
        _check_records(info, mat["inst_map"], im, mat["raw_map"])
        uid = mat["inst_uid"].ravel()
        want = np.array([[info[int(i)]["features"][n] for n in _lib.FEATURE_NAMES] for i in uid])
        assert np.array_equal(mat["inst_features"], want)
        # without save_raw_map the prediction map stays on the device for np_prob_mean: the same records
        assert json.load(open(str(tmp_path / "plain" / "json" / ("%s.json" % k))))["nuc"] == js
        off = json.load(open(str(tmp_path / "off" / "json" / ("%s.json" % k))))["nuc"]
        assert off == {i: {kk: vv for kk, vv in v.items() if kk != "features"} for i, v in js.items()}
        assert "inst_features" not in sio.loadmat(str(tmp_path / "off" / "mat" / ("%s.mat" % k)))
    mgr.net.ctx.close()


def test_cli_wsi_save_features(tmp_path):
    """`run_infer.py ... wsi --save_features` on the small synthetic slide: every record's features are the
    restatement on its pixels in the written instance map, the slide and the prediction map."""
    import cv2
    from hover_net_b200 import run_infer, synth
    from hover_net_b200.infer import wsi
    h, w = 600, 700
    base = synth.make_patches(12, 256, seed=60)
    img = np.concatenate([np.concatenate(list(base[r * 3:(r + 1) * 3]), 1) for r in range(3)], 0)[:h, :w].copy()
    os.makedirs(tmp_path / "in")
    np.save(str(tmp_path / "in" / "slide.npy"), img)
    np.savez(str(tmp_path / "ckpt.npz"), **synth.make_state_dict("fast", 6, seed=0))
    os.makedirs(tmp_path / "msk")
    cv2.imwrite(str(tmp_path / "msk" / "slide.png"), np.full((h // 8, w // 8), 255, np.uint8))
    argv = ["--nr_types=6", "--model_mode=fast", "--model_path=%s" % (tmp_path / "ckpt.npz"), "--batch_size=8", "wsi",
            "--input_dir=%s" % (tmp_path / "in"), "--output_dir=%s" % (tmp_path / "out"),
            "--cache_path=%s" % (tmp_path / "cache"), "--input_mask_dir=%s" % (tmp_path / "msk"), "--chunk_shape=500",
            "--tile_shape=256", "--ambiguous_size=32", "--save_features"]
    cmd, margs, rargs, _ = run_infer.parse(argv)
    margs["method"]["model_args"]["device"] = 0
    mgr = wsi.InferManager(**margs)
    mgr.process_wsi_list(rargs)
    js = json.load(open(str(tmp_path / "out" / "slide.json")))["nuc"]
    _check_records({int(k): v for k, v in js.items()}, mgr.wsi_inst_map, img, np.array(mgr.wsi_pred_map))
    mgr.net.ctx.close()
