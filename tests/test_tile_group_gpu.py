"""Tile groups (`hvn_infer_tiles`): many images of any sizes through one stream of patch batches, post-processed per
size class, must give every image exactly what the single-image path gives it."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SHAPES = [(256, 256), (300, 420), (1000, 1000), (100, 80), (30, 300), (256, 256)]  # the 2nd 256^2 makes slot != input order
GEOM = {"fast": (256, 164), "original": (270, 80)}


def _img(h, w, seed):
    from hover_net_b200 import synth
    k = -(-max(h, w) // 256)
    tiles = synth.make_patches(k * k, 256, seed=seed)
    big = np.concatenate([np.concatenate(list(tiles[r * k:(r + 1) * k]), 1) for r in range(k)], 0)
    return np.ascontiguousarray(big[:h, :w])


def _manager(mode, nt, sd=None):
    from hover_net_b200 import synth
    from hover_net_b200.infer.tile import InferManager
    mgr = InferManager(method={"model_args": {"nr_types": nt, "mode": mode},
                               "model_path": sd if sd is not None else synth.make_state_dict(mode, nt, seed=0)},
                       type_info_path=None)
    mgr.patch_input_shape, mgr.patch_output_shape = GEOM[mode]
    return mgr


def _same_result(a, b):
    (pa, ia, da), (pb, ib, db) = a, b
    assert pa.shape == pb.shape and np.array_equal(pa.view(np.uint32), pb.view(np.uint32))
    assert ia.dtype == ib.dtype and np.array_equal(ia, ib)
    assert list(da.keys()) == list(db.keys())
    for k in da:
        x, y = da[k], db[k]
        assert np.array_equal(x["bbox"], y["bbox"]) and np.array_equal(x["centroid"], y["centroid"])
        assert np.array_equal(x["contour"], y["contour"]) and x["contour"].dtype == y["contour"].dtype
        assert x["type"] == y["type"] and x["type_prob"] == y["type_prob"]


def test_range_retry_in_group():
    """A checkpoint whose activations leave the fp16 range: the reference's raw initialisation (net_utils.py:18-32, as
    in test_cnn_gpu.py::test_reference_weights_init_checkpoint) with the stem scaled by 3e5, as in
    test_cnn_gpu.py::test_range_overflow_is_an_error_not_a_clamp.  The raw initialisation alone stays within the range
    on these images at act_shift 0, so it would not exercise the retry.  A group raises act_shift in one call to what
    the per-image path needs, and then equals the per-image path at that act_shift."""
    from hover_net_b200 import synth
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
    sd["conv0./.weight"] = (sd["conv0./.weight"] * np.float32(3.0e5)).astype(np.float32)
    imgs = [synth.make_patches(1, 256, seed=33)[0], _img(100, 80, 31), _img(300, 420, 32), _img(1000, 1000, 33),
            _img(512, 512, 34)]
    a, b = _manager(mode, nt, sd), _manager(mode, nt, sd)
    try:
        singles = [b.net.ctx.infer_tile(img, 256, 5) for img in imgs]   # raises b's act_shift as far as any image needs
        need = b.net.ctx.counter("act_shift")
        assert need > 0, "no image of this group leaves the fp16 range"
        assert a.net.ctx.counter("act_shift") == 0
        group = a.net.ctx.infer_tiles(imgs, 256, 5)
        assert a.net.ctx.counter("act_shift") == need
        # b's early images ran below `need`; rerun them at the same act_shift
        singles = [b.net.ctx.infer_tile(img, 256, 5) for img in imgs]
        assert b.net.ctx.counter("act_shift") == need
        for g, one in zip(group, singles):
            assert np.array_equal(g[0], one[0]) and np.array_equal(g[1], one[1]) and np.array_equal(g[2], one[2])
            assert np.array_equal(g[4], one[4]) and np.array_equal(g[3], one[3][: len(g[3])])
    finally:
        a.net.ctx.close()
        b.net.ctx.close()


def test_mixed_group_tables_scale_with_each_image():
    """Each image's padded instance table holds min(rows_cap, H*W/6 + 8) rows of its own size, not the largest
    image's: the workspace of a mixed group follows its pixels."""
    from hover_net_b200 import _lib
    mgr = _manager("fast", 6)
    ctx = mgr.net.ctx
    try:
        shapes = [(64, 64)] * 4 + [(1000, 1000)] + [(64, 64)] * 4 + [(30, 300)]
        imgs = [_img(h, w, 130 + i) for i, (h, w) in enumerate(shapes)]
        rows_cap, _ = _lib.tiles_sizes(np.array(shapes))
        got = ctx.infer_tiles(imgs, 256, 16)
        want_rows = sum(min(rows_cap, h * w // 6 + 8) for h, w in shapes)
        assert ctx.counter("tile_table_rows") == want_rows < len(shapes) * min(rows_cap, 1000 * 1000 // 6 + 8) // 5
        from hover_net_b200.infer import tile
        for (h, w) in shapes:  # the planner charges at least the table workspace of every image
            assert tile._file_cost((h, w, 3), 256, 164)[1] >= 84 * (h * w // 6 + 8) + 24 * h * w
        for g, img in zip(got, imgs):
            one = ctx.infer_tile(img, 256, 16)
            assert np.array_equal(g[1], one[1]) and np.array_equal(g[2], one[2]) and np.array_equal(g[4], one[4])
    finally:
        ctx.close()


def _raw_tiles(ctx, imgs, rows_cap, pts_cap, batch=8):
    from hover_net_b200 import _lib
    packed, shapes = _lib.pack_images(imgs)
    px = packed.size // 3
    inst = np.empty((px,), np.int32)
    table = np.zeros((rows_cap, 10), np.int64)
    ro = np.zeros((len(imgs) + 1,), np.int32)
    po = np.zeros((rows_cap + 1,), np.int32)
    pts = np.zeros((max(pts_cap, 1), 2), np.int32)
    L = _lib.lib()
    L.hvn_infer_tiles.argtypes = _lib._TILES_ARGS
    rc = L.hvn_infer_tiles(ctx._h, len(imgs), _lib._ptr(packed), _lib._ptr(shapes), 256, batch, None, _lib._ptr(inst),
                           _lib._ptr(table), rows_cap, _lib._ptr(ro), _lib._ptr(pts), pts_cap, _lib._ptr(po))
    return rc, inst, table, ro, po, pts


def test_capacity_retries():
    mgr = _manager("fast", 6)
    ctx = mgr.net.ctx
    try:
        imgs = [_img(h, w, 50 + i) for i, (h, w) in enumerate([(300, 420), (256, 256), (100, 80), (300, 420)])]
        want = ctx.infer_tiles(imgs, 256, 8)
        rows = sum(len(w[2]) for w in want)
        npts = sum(len(w[4]) for w in want)
        assert rows > 4 and npts > 4
        rc, _, _, ro, _, _ = _raw_tiles(ctx, imgs, 2, 1)
        assert rc == -4 and int(ro[-1]) == rows                      # the table: exact size reported
        rc, _, _, ro, po, _ = _raw_tiles(ctx, imgs, rows, 3)
        assert rc == -4 and int(po[rows]) == npts                    # the points: exact size reported
        rc, inst, table, ro, po, pts = _raw_tiles(ctx, imgs, rows, npts)
        assert rc == 0
        from hover_net_b200 import _lib
        got = _lib.split_tiles(np.array([i.shape[:2] for i in imgs]), inst, table, ro, None, pts[:npts], po[:rows + 1])
        for g, w in zip(got, want):
            for x, y in zip(g[1:], w[1:]):
                assert np.array_equal(x, y)
        small = ctx.infer_tiles(imgs, 256, 8, rows_cap=1, pts_cap=1)  # the binding's retries end at the same result
        for g, w in zip(small, want):
            for x, y in zip(g, w):
                assert np.array_equal(x, y)
        assert ctx.infer_tiles([imgs[2]], 256, 8, rows_cap=1, pts_cap=0)[0][1].shape == (100, 80)
    finally:
        ctx.close()


def test_bad_arguments():
    from hover_net_b200 import _lib
    mgr = _manager("fast", 6)
    ctx = mgr.net.ctx
    try:
        img = np.zeros((10, 10, 3), np.uint8)
        L = _lib.lib()
        L.hvn_infer_tiles.argtypes = _lib._TILES_ARGS
        inst, table, ro = np.empty(100, np.int32), np.empty((16, 10), np.int64), np.empty(2, np.int32)
        for n, shapes, cap in [(0, np.array([[10, 10]], np.int32), 16), (1, np.array([[0, 10]], np.int32), 16),
                               (1, np.array([[10, 10]], np.int32), 0)]:
            rc = L.hvn_infer_tiles(ctx._h, n, _lib._ptr(img), _lib._ptr(shapes), 256, 4, None, _lib._ptr(inst),
                                   _lib._ptr(table), cap, _lib._ptr(ro), None, 0, None)
            assert rc == -1
    finally:
        ctx.close()


def test_dev_variant_is_stream_ordered():
    from hover_net_b200 import _lib
    mgr = _manager("fast", 6)
    ctx = mgr.net.ctx
    try:
        imgs = [_img(h, w, 70 + i) for i, (h, w) in enumerate([(256, 256), (300, 420), (256, 256), (30, 300)])]
        want = ctx.infer_tiles(imgs, 256, 7)
        packed, shapes = _lib.pack_images(imgs)
        px = packed.size // 3
        rows_cap, pts_cap = _lib.tiles_sizes(shapes)
        sizes = dict(img=packed.nbytes, pred=px * 16, inst=px * 4, table=rows_cap * 80, ro=(len(imgs) + 1) * 4,
                     po=(rows_cap + 1) * 4, pts=pts_cap * 8)
        d = {k: ctx.malloc(b) for k, b in sizes.items()}
        try:
            ctx.h2d(d["img"], packed, packed.nbytes)
            ctx.infer_tiles_dev(len(imgs), d["img"], shapes, 256, 7, d["pred"], d["inst"], d["table"], rows_cap, d["ro"],
                                d["pts"], pts_cap, d["po"])
            ctx.sync()
            ro = np.empty((len(imgs) + 1,), np.int32)
            ctx.d2h(ro, d["ro"], ro.nbytes)
            rows = int(ro[-1])
            po = np.empty((rows + 1,), np.int32)
            ctx.d2h(po, d["po"], po.nbytes)
            pred, inst = np.empty((px * 4,), np.float32), np.empty((px,), np.int32)
            table, pts = np.empty((rows, 10), np.int64), np.empty((int(po[-1]), 2), np.int32)
            for a, k in [(pred, "pred"), (inst, "inst"), (table, "table"), (pts, "pts")]:
                ctx.d2h(a, d[k], a.nbytes)
            ctx.sync()
        finally:
            for p in d.values():
                ctx.free(p)
        got = _lib.split_tiles(shapes, inst, table, ro, pred, pts, po)
        for g, w in zip(got, want):
            for x, y in zip(g, w):
                assert np.array_equal(x, y)
        job = ctx.infer_tiles_begin(imgs, 256, 7, want_pred=False)
        for g, w in zip(job.result(), want):
            assert g[0] is None
            for x, y in zip(g[1:], w[1:]):
                assert np.array_equal(x, y)
    finally:
        ctx.close()


def test_process_file_list_grouped_equals_one_file_at_a_time(tmp_path):
    """12 mixed images: groups of one (tiny mem_usage) and one group write the same files.  A .mat header carries its
    creation time, so .mat files are compared after the 116-byte header text."""
    import cv2
    os.makedirs(tmp_path / "in")
    shapes = [(256, 256), (300, 420), (256, 256), (100, 80), (512, 300), (256, 256), (30, 300), (300, 420),
              (256, 256), (164, 164), (256, 256), (400, 256)]
    for i, (h, w) in enumerate(shapes):
        cv2.imwrite(str(tmp_path / "in" / ("f%02d.png" % i)), cv2.cvtColor(_img(h, w, 90 + i), cv2.COLOR_RGB2BGR))
    mgr = _manager("fast", 6)
    outs = {}
    try:
        for name, mem in [("single", 1e-12), ("grouped", 0.5)]:
            out = tmp_path / name
            mgr.process_file_list({"batch_size": 16, "nr_inference_workers": 0, "nr_post_proc_workers": 0,
                                   "patch_input_shape": 256, "patch_output_shape": 164, "input_dir": str(tmp_path / "in"),
                                   "output_dir": str(out), "mem_usage": mem, "draw_dot": True, "save_qupath": True,
                                   "save_raw_map": True})
            outs[name] = out
    finally:
        mgr.net.ctx.close()
    n = 0
    for sub, ext in [("mat", ".mat"), ("json", ".json"), ("qupath", ".tsv"), ("overlay", ".png")]:
        a = sorted(os.listdir(outs["single"] / sub))
        assert a == sorted(os.listdir(outs["grouped"] / sub)) and len(a) == 12
        for f in a:
            x = open(outs["single"] / sub / f, "rb").read()
            y = open(outs["grouped"] / sub / f, "rb").read()
            skip = 116 if ext == ".mat" else 0
            assert x[skip:] == y[skip:], f
            n += 1
    assert n == 48


def test_grouping_follows_the_ram_budget(monkeypatch):
    """One group under the default budget, groups of one under a tiny one (the planner, not the device, decides)."""
    from hover_net_b200.infer import tile
    seen = []
    real = tile._groups

    def spy(items, costs, budgets):
        for g in real(items, costs, budgets):
            seen.append(len(g))
            yield g
    monkeypatch.setattr(tile, "_groups", spy)
    import cv2
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, "in"))
        for i in range(3):
            cv2.imwrite(os.path.join(d, "in", "g%d.png" % i), _img(200, 200, i))
        mgr = _manager("fast", 6)
        try:
            for mem in (1e-12, 0.5):
                mgr.process_file_list({"patch_input_shape": 256, "patch_output_shape": 164, "input_dir": d + "/in",
                                       "output_dir": d + "/out", "mem_usage": mem})
        finally:
            mgr.net.ctx.close()
    assert seen == [1, 1, 1, 3]


def _two_rank_group_worker(rank, world, port, out):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from hover_net_b200 import synth
    from hover_net_b200.infer.tile import InferManager
    mode, nt = "fast", 6
    mgr = InferManager(method={"model_args": {"nr_types": nt, "mode": mode, "device": rank},
                               "model_path": synth.make_state_dict(mode, nt, seed=0)}, type_info_path=None)
    mgr.patch_input_shape, mgr.patch_output_shape, mgr.batch_size = 256, 164, 4
    imgs = [_img(h, w, 110 + i) for i, (h, w) in enumerate([(300, 420), (256, 256), (100, 80), (500, 610)])]
    from hover_net_b200.models.hovernet.post_proc import table_to_dict
    group = mgr.infer_images(imgs, all_ranks=True)          # combined patch list sharded over the ranks + all_reduce
    one = [(p, i, table_to_dict(t, o, pts, nt)) for p, i, t, o, pts in mgr.net.ctx.infer_tiles(imgs, 256, 4)]
    ok = True                                               # the same group on this rank alone
    for g, o in zip(group, one):
        try:
            _same_result(g, o)
        except AssertionError:
            ok = False
    ok = ok and sum(len(g[2]) for g in group) > 0
    flags = [None] * world
    dist.all_gather_object(flags, ok)
    if rank == 0:
        out.put(flags)
    dist.barrier()
    mgr.net.ctx.close()
    dist.destroy_process_group()


def test_group_sharded_over_two_gpus_equals_single_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_two_rank_group_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    flags = q.get(timeout=600)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert flags == [True, True]


# Last in the module: the contexts of this fixture live until the module ends, with the plans of every batch tail.
@pytest.fixture(scope="module", params=[("fast", 6), ("original", 5)], ids=["fast6", "original5"])
def setup(request):
    mode, nt = request.param
    mgr = _manager(mode, nt)
    imgs = [_img(h, w, 10 + i) for i, (h, w) in enumerate(SHAPES)]
    mgr.batch_size = 32
    singles = [mgr.infer_image(img) for img in imgs]
    assert sum(len(s[2]) for s in singles) > 0
    yield mode, nt, mgr, imgs, singles
    mgr.net.ctx.close()


@pytest.mark.parametrize("batch", [3, 32, 125])
def test_mixed_group_equals_single_images(setup, batch):
    mode, nt, mgr, imgs, singles = setup
    ctx = mgr.net.ctx
    cells = np.cumsum([0] + [np.prod(ctx.tile_grid(h, w, GEOM[mode][0])) for h, w in SHAPES])
    # batches are cut from one patch list: some batch holds patches of two images
    assert any(len({int(np.searchsorted(cells, p, "right")) for p in range(b, min(b + batch, cells[-1]))}) > 1
               for b in range(0, int(cells[-1]), batch))
    mgr.batch_size = batch
    try:
        group = mgr.infer_images(imgs)
    finally:
        mgr.batch_size = 32
    assert len(group) == len(imgs)
    for g, s in zip(group, singles):
        _same_result(g, s)
