"""Host-buffer entry points against their device-pointer twins, and the guarantees of the host staging.

* Every host call gives bit-identical outputs to the same work through the `_dev` entry points (or, for hvn_infer_tile,
  through hvn_infer_tiles on a group of one), fast mode, 256 x 256 patches, B = 2, nr_types 6 and None; the tile group
  is 200x300, 300x200, 200x300, so equal sizes are grouped and the slot order is not the input order.
* Through the raw C ABI with host buffers pre-filled with -1: padded table rows past n_rows come back as zeros; on
  HVN_ERR_CAPACITY the row counts / offsets report the exact sizes and no point past the capacity is written.
* A range overflow is reported before a capacity failure (the binding's act_shift retry depends on it).
Raw calls pass int64_t arguments as c_int64 and pointers through _lib._ptr, so they do not depend on the prototypes."""
import ctypes

import numpy as np
import pytest

from hover_net_b200 import synth

pytestmark = pytest.mark.gpu

I64 = ctypes.c_int64
B, S, OUT = 2, 256, 164
TILE_SHAPES = [(200, 300), (300, 200), (200, 300)]


def _net(nt, sd=None):
    from hover_net_b200.models.hovernet.net_desc import create_model
    net = create_model(mode="fast", input_ch=3, nr_types=nt)
    net.load_state_dict(sd if sd is not None else synth.make_state_dict("fast", nt, seed=0), strict=True)
    return net


@pytest.fixture(scope="module", params=[6, None], ids=["nt6", "ntNone"])
def net(request):
    n = _net(request.param)
    yield n
    n.ctx.close()


class _Dev:
    """Device copies of host arrays on one context, freed at the end."""

    def __init__(self, ctx):
        self.ctx, self.ptrs = ctx, []

    def empty(self, nbytes):
        p = self.ctx.malloc(max(int(nbytes), 1))
        self.ptrs.append(p)
        return p

    def put(self, a):
        a = np.ascontiguousarray(a)
        p = self.empty(a.nbytes)
        self.ctx.h2d(p, a, a.nbytes)
        return p

    def get(self, p, shape, dtype):
        a = np.empty(shape, dtype)
        self.ctx.d2h(a, p, a.nbytes)
        self.ctx.sync()
        return a

    def free(self):
        self.ctx.sync()
        for p in self.ptrs:
            self.ctx.free(p)


@pytest.fixture
def dev(net):
    d = _Dev(net.ctx)
    yield d
    d.free()


def _same(a, b):
    if a is None or b is None:
        assert a is None and b is None
        return
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _nt(net):
    return int(net.ctx.nr_types or 0)


def _pred_maps(net, seed=0):
    C = 4 if _nt(net) else 3
    return np.stack([synth.synth_pred_map(OUT, OUT, net.ctx.nr_types, seed=seed + i)[..., -C:] for i in range(B)])


def _tile_imgs():
    out = []
    for i, (h, w) in enumerate(TILE_SHAPES):
        x = synth.make_patches(4, S, seed=50 + i)
        big = np.concatenate([np.concatenate(list(x[:2]), 1), np.concatenate(list(x[2:]), 1)], 0)
        out.append(np.ascontiguousarray(big[:h, :w]))
    return out


def _labels(nt, seed=11):
    imgs = synth.make_patches(B, S, seed=seed)
    inst = np.stack([synth.synth_instances(S, S, seed=seed * 10 + i) for i in range(B)]).astype(np.int32)
    typ = np.where(inst > 0, inst % nt, 0).astype(np.int32) if nt else None
    return imgs, inst, typ


# ---- host call == device twin ----------------------------------------------------------------------------------------
def test_forward(net, dev):
    x = synth.make_patches(B, S, seed=1)
    host = net.ctx.forward(x)
    d_out = dev.empty(host.nbytes)
    net.ctx.forward_dev(dev.put(x), B, S, S, d_out)
    _same(host, dev.get(d_out, host.shape, np.float32))


def _postproc_dev(net, dev, pred, max_rows):
    n, H, W, C = pred.shape
    d_inst, d_tab, d_nr = dev.empty(n * H * W * 4), dev.put(np.zeros((n, max_rows, 10), np.int64)), dev.empty(n * 4)
    net.ctx.postproc_dev(dev.put(pred), n, H, W, C, net.ctx.nr_types, d_inst, d_tab, max_rows, d_nr)
    nr = dev.get(d_nr, (n,), np.int32)
    return (dev.get(d_inst, (n, H, W), np.int32), dev.get(d_tab, (n, max_rows, 10), np.int64), nr), (d_inst, d_tab, d_nr)


def test_postproc(net, dev):
    pred = _pred_maps(net)
    inst, table, nrows = net.ctx.postproc(pred, net.ctx.nr_types, max_rows=400)
    (di, dt, dn), _ = _postproc_dev(net, dev, pred, 400)
    _same(inst, di), _same(nrows, dn), _same(table, dt)
    assert nrows.min() > 0


def test_postproc_contours(net, dev):
    pred = _pred_maps(net, seed=3)
    n, H, W, _ = pred.shape
    inst, table, nrows, offs, pts = net.ctx.postproc_contours(pred, net.ctx.nr_types, max_rows=400, pts_cap=1 << 16)
    (di, dt, dn), (d_inst, d_tab, d_nr) = _postproc_dev(net, dev, pred, 400)
    cap = 1 << 16
    d_pts, d_offs = dev.empty(cap * 8), dev.empty((n * 400 + 1) * 4)
    net.ctx.contours_dev(d_inst, d_tab, d_nr, n, H, W, 400, d_pts, cap, d_offs)
    doffs = dev.get(d_offs, (n * 400 + 1,), np.int32)
    _same(inst, di), _same(nrows, dn), _same(table, dt), _same(offs, doffs)
    _same(pts, dev.get(d_pts, (int(doffs[-1]), 2), np.int32))
    assert len(pts) > 0


@pytest.mark.parametrize("want_pred", [True, False])
def test_forward_postproc(net, dev, want_pred):
    x = synth.make_patches(B, S, seed=2)
    pred, inst, table, nrows = net.ctx.forward_postproc(x, want_pred=want_pred, max_rows=300)
    C = 4 if _nt(net) else 3
    d_pred = dev.empty(B * OUT * OUT * C * 4) if want_pred else None
    d_inst, d_tab, d_nr = dev.empty(B * OUT * OUT * 4), dev.put(np.zeros((B, 300, 10), np.int64)), dev.empty(B * 4)
    net.ctx.forward_postproc_dev(dev.put(x), B, S, S, d_pred, d_inst, d_tab, 300, d_nr)
    _same(inst, dev.get(d_inst, (B, OUT, OUT), np.int32))
    _same(nrows, dev.get(d_nr, (B,), np.int32))
    _same(table, dev.get(d_tab, (B, 300, 10), np.int64))
    _same(pred, dev.get(d_pred, (B, OUT, OUT, C), np.float32) if want_pred else None)


def test_infer_tiles(net, dev):
    from hover_net_b200 import _lib
    imgs = _tile_imgs()
    host = net.ctx.infer_tiles(imgs, S, batch=4)
    packed, shapes = _lib.pack_images(imgs)
    n, px, C = len(imgs), packed.size // 3, 4 if _nt(net) else 3
    rows_cap, pts_cap = _lib.tiles_sizes(shapes)
    d = [dev.empty(b) for b in (px * C * 4, px * 4, rows_cap * 80, (n + 1) * 4, pts_cap * 8, (rows_cap + 1) * 4)]
    net.ctx.infer_tiles_dev(n, dev.put(packed), shapes, S, 4, *d[:3], rows_cap, d[3], d[4], pts_cap, d[5])
    ro = dev.get(d[3], (n + 1,), np.int32)
    rows = int(ro[-1])
    po = dev.get(d[5], (rows_cap + 1,), np.int32)[: rows + 1]
    out = _lib.split_tiles(shapes, dev.get(d[1], (px,), np.int32), dev.get(d[2], (rows_cap, 10), np.int64)[:rows], ro,
                           dev.get(d[0], (px * C,), np.float32), dev.get(d[4], (int(po[-1]), 2), np.int32), po)
    assert len(host) == len(out) == n and rows > 0
    for h, o in zip(host, out):
        for a, b in zip(h, o):
            _same(a, b)


def test_infer_tile_equals_group_of_one(net):
    img = _tile_imgs()[1]
    pred, inst, table, offs, pts = net.ctx.infer_tile(img, S, 4)
    (grp,) = net.ctx.infer_tiles([img], S, batch=4)
    _same(pred, grp[0]), _same(inst, grp[1]), _same(table, grp[2]), _same(pts, grp[4])
    _same(offs[: len(table) + 1].astype(np.int64), grp[3])
    assert len(table) > 0


def test_inst_pairs(net, dev):
    _, t, _ = _labels(5, seed=12)
    _, p, _ = _labels(5, seed=13)
    rows, offs = net.ctx.inst_pairs(t, p)
    n, H, W = t.shape
    total = int(offs[-1])
    d_pairs, d_offs = dev.empty(total * 24), dev.empty((n + 1) * 8)
    assert net.ctx.inst_pairs_dev(dev.put(t), dev.put(p), n, H, W, d_pairs, total, d_offs)
    doffs = dev.get(d_offs, (n + 1,), np.int64)
    drows = dev.get(d_pairs, (total, 3), np.int64)
    m = np.repeat(np.arange(n), np.diff(doffs))
    _same(offs, doffs), _same(rows, drows[np.lexsort((drows[:, 1], drows[:, 0], m))])


def test_targets(net, dev):
    _, inst, _ = _labels(0, seed=14)
    hv, flags = net.ctx.targets(inst, (OUT, OUT))
    n, H, W = inst.shape
    d_hv, d_flags = dev.empty(hv.nbytes), dev.empty(flags.nbytes)
    net.ctx.targets_dev(dev.put(inst), n, H, W, OUT, OUT, d_hv, d_flags)
    _same(hv, dev.get(d_hv, hv.shape, np.float32)), _same(flags, dev.get(d_flags, flags.shape, np.int32))


def _valid_dev_bufs(net, dev):
    nt = _nt(net)
    return dev.empty((3 + 2 * nt) * 8), dev.empty(8), dev.empty(B * 4)


def test_valid(net, dev):
    nt = _nt(net)
    imgs, inst, typ = _labels(nt, seed=15)
    counts, sse, flags = net.ctx.valid(imgs, inst, typ)
    d_c, d_s, d_f = _valid_dev_bufs(net, dev)
    net.ctx.valid_dev(dev.put(imgs), dev.put(inst), dev.put(typ) if nt else None, B, S, S, d_c, d_s, d_f)
    _same(counts, dev.get(d_c, counts.shape, np.int64)), _same(flags, dev.get(d_f, (B,), np.int32))
    # hvn_valid's hv_sse is an fp64 atomic sum: equal from call to call up to the order of the additions
    assert abs(dev.get(d_s, (1,), np.float64)[0] - sse) <= 1e-12 * sse


@pytest.mark.parametrize("want_probs", [True, False])
def test_valid_loss(net, dev, want_probs):
    nt = _nt(net)
    imgs, inst, typ = _labels(nt, seed=16)
    counts, sse, flags, sums, probs = net.ctx.valid_loss(imgs, inst, typ, want_probs=want_probs)
    d_c, d_s, d_f = _valid_dev_bufs(net, dev)
    d_sums = dev.empty(sums.nbytes)
    d_probs = dev.empty(B * OUT * OUT * (4 + nt) * 4) if want_probs else None
    net.ctx.valid_loss_dev(dev.put(imgs), dev.put(inst), dev.put(typ) if nt else None, B, S, S, d_c, d_s, d_f, d_sums,
                           d_probs)
    _same(counts, dev.get(d_c, counts.shape, np.int64))
    _same(np.float64(sse), dev.get(d_s, (1,), np.float64)[0]), _same(flags, dev.get(d_f, (B,), np.int32))
    _same(sums, dev.get(d_sums, sums.shape, np.float64))
    _same(probs, dev.get(d_probs, (B, OUT, OUT, 4 + nt), np.float32) if want_probs else None)


# ---- raw ABI: zeroed padding, exact sizes on HVN_ERR_CAPACITY ---------------------------------------------------------
def _sentinel(shape, dtype):
    return np.full(shape, -1, dtype)


def _raw():
    from hover_net_b200 import _lib
    return _lib.lib(), _lib._ptr


def test_padded_rows_come_back_as_zeros(net):
    L, p = _raw()
    h, nt = net.ctx._h, _nt(net)
    pred = _pred_maps(net, seed=7)
    n, H, W, C = pred.shape
    M = 400

    def bufs(nm, hh, ww):
        return _sentinel((nm, hh, ww), np.int32), _sentinel((nm, M, 10), np.int64), _sentinel((nm,), np.int32)

    inst, tab, nr = bufs(n, H, W)
    assert L.hvn_postproc(h, p(pred), n, H, W, C, nt, p(inst), p(tab), M, p(nr)) == 0
    tables = [(tab, nr)]
    inst, tab, nr = bufs(n, H, W)
    offs, pts = _sentinel((n * M + 1,), np.int32), _sentinel((1 << 16, 2), np.int32)
    assert L.hvn_postproc_contours(h, p(pred), n, H, W, C, nt, p(inst), p(tab), M, p(nr), p(pts), I64(1 << 16),
                                   p(offs)) == 0
    tables.append((tab, nr))
    x = synth.make_patches(B, S, seed=8)
    inst, tab, nr = bufs(B, OUT, OUT)
    assert L.hvn_forward_postproc(h, p(x), B, S, S, None, p(inst), p(tab), M, p(nr)) == 0
    tables.append((tab, nr))
    img = _tile_imgs()[0]
    inst, tab, nr = bufs(1, *img.shape[:2])
    offs, pts = _sentinel((M + 1,), np.int32), _sentinel((1 << 16, 2), np.int32)
    assert L.hvn_infer_tile(h, p(img), img.shape[0], img.shape[1], S, 4, None, p(inst), p(tab[0]), M, p(nr), p(pts),
                            I64(1 << 16), p(offs)) == 0
    tables.append((tab, nr))
    for tab, nr in tables:
        for m in range(len(nr)):
            k = int(nr[m])
            assert k < M and (tab[m, :k, 0] > 0).all() and not tab[m, k:].any()


def test_capacity_reports_exact_sizes(net):
    L, p = _raw()
    h, nt = net.ctx._h, _nt(net)
    pred = _pred_maps(net, seed=9)
    n, H, W, C = pred.shape
    _, _, ref_nr, ref_offs, ref_pts = net.ctx.postproc_contours(pred, net.ctx.nr_types, max_rows=400, pts_cap=1 << 16)
    total = len(ref_pts)
    # the table too small: hvn_postproc reports every map's row count
    inst, tab, nr = _sentinel((n, H, W), np.int32), _sentinel((n, 1, 10), np.int64), _sentinel((n,), np.int32)
    assert L.hvn_postproc(h, p(pred), n, H, W, C, nt, p(inst), p(tab), 1, p(nr)) == -4
    _same(nr, ref_nr)
    # the point buffer too small: offsets exact, nothing written past the capacity
    cap = total // 2
    inst, tab, nr = _sentinel((n, H, W), np.int32), _sentinel((n, 400, 10), np.int64), _sentinel((n,), np.int32)
    offs, pts = _sentinel((n * 400 + 1,), np.int32), _sentinel((total, 2), np.int32)
    assert L.hvn_postproc_contours(h, p(pred), n, H, W, C, nt, p(inst), p(tab), 400, p(nr), p(pts), I64(cap),
                                   p(offs)) == -4
    _same(offs, ref_offs), _same(nr, ref_nr)
    assert (pts[cap:] == -1).all()

    from hover_net_b200 import _lib
    imgs = _tile_imgs()
    ref = net.ctx.infer_tiles(imgs, S, batch=4, want_pred=False)
    img = imgs[int(np.argmax([len(r[2]) for r in ref]))]
    Hi, Wi = img.shape[:2]
    _, _, ref_tab, ref_offs, ref_pts = net.ctx.infer_tile(img, S, 4, want_pred=False)
    rows, total = len(ref_tab), len(ref_pts)
    assert rows >= 2 and total >= 2
    inst, nr = _sentinel((Hi, Wi), np.int32), _sentinel((1,), np.int32)
    tab, offs, pts = _sentinel((1, 10), np.int64), _sentinel((2,), np.int32), _sentinel((total, 2), np.int32)
    assert L.hvn_infer_tile(h, p(img), Hi, Wi, S, 4, None, p(inst), p(tab), 1, p(nr), p(pts), I64(total), p(offs)) == -4
    assert int(nr[0]) == rows
    M, cap = rows + 5, total // 2
    tab, offs = _sentinel((M, 10), np.int64), _sentinel((M + 1,), np.int32)
    assert L.hvn_infer_tile(h, p(img), Hi, Wi, S, 4, None, p(inst), p(tab), M, p(nr), p(pts), I64(cap), p(offs)) == -4
    _same(offs[: rows + 1], ref_offs[: rows + 1])
    assert int(offs[-1]) == total and (pts[cap:] == -1).all()

    packed, shapes = _lib.pack_images(imgs)
    px = packed.size // 3
    ref_ro = np.cumsum([0] + [len(r[2]) for r in ref]).astype(np.int32)
    rows, total = int(ref_ro[-1]), sum(len(r[4]) for r in ref)
    inst = _sentinel((px,), np.int32)
    for rows_cap, pts_cap in ((1, total), (rows, total // 2)):
        tab, ro = _sentinel((rows_cap, 10), np.int64), _sentinel((len(imgs) + 1,), np.int32)
        po, pts = _sentinel((rows_cap + 1,), np.int32), _sentinel((total, 2), np.int32)
        assert L.hvn_infer_tiles(h, len(imgs), p(packed), p(shapes), S, 4, None, p(inst), p(tab), I64(rows_cap), p(ro),
                                 p(pts), I64(pts_cap), p(po)) == -4
        _same(ro, ref_ro)
        if rows_cap == rows:
            assert int(po[rows]) == total and (pts[pts_cap:] == -1).all()
        else:
            assert (tab == -1).all()

    _, t, _ = _labels(5, seed=12)
    ref_rows, ref_offs = net.ctx.inst_pairs(t)
    pairs, offs = _sentinel((4, 3), np.int64), _sentinel((B + 1,), np.int64)
    assert L.hvn_inst_pairs(h, p(t), None, B, S, S, p(pairs), I64(1), p(offs)) == -4
    _same(offs, ref_offs)
    assert (pairs == -1).all()


def test_range_error_before_capacity_error():
    L, p = _raw()
    sd = dict(synth.make_state_dict("fast", 6, seed=0))
    sd["conv0./.weight"] = (sd["conv0./.weight"] * np.float32(3.0e5)).astype(np.float32)
    sd["conv0.bn.running_var"] = np.full_like(sd["conv0.bn.running_var"], 1.0)
    net = _net(6, sd=sd)
    try:
        x = synth.make_patches(B, S, seed=3)
        inst, tab, nr = np.empty((B, OUT, OUT), np.int32), np.zeros((B, 1, 10), np.int64), np.zeros((B,), np.int32)
        rc = L.hvn_forward_postproc(net.ctx._h, p(x), B, S, S, None, p(inst), p(tab), 1, p(nr))
        assert rc == -6 and b"act_shift" in L.hvn_last_error()
    finally:
        net.ctx.close()
