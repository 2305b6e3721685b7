"""Host side of tile groups: the file-grouping rule of `process_file_list` and the helpers that pack a group's images
and split its packed outputs back into per-image arrays."""
import sys

import numpy as np

from hover_net_b200 import _lib
from hover_net_b200.infer import tile


def _cut(costs, budgets):
    """Groups of indices for items with the given (ram, dev) costs; budgets is a list, one entry per group."""
    it = iter(budgets)
    return [[i for i, _ in g] for g in tile._groups(list(enumerate(costs)), lambda x: x[1], lambda: next(it))]


def test_groups_keep_file_order_and_fill_the_budget():
    costs = [(3, 0), (4, 0), (2, 0), (5, 0), (1, 0)]
    assert _cut(costs, [(9, None)] * 5) == [[0, 1, 2], [3, 4]]
    assert _cut(costs, [(100, None)]) == [[0, 1, 2, 3, 4]]
    # the budget is read afresh for every group
    assert _cut(costs, [(3, None), (6, None), (100, None)]) == [[0], [1, 2], [3, 4]]


def test_file_over_budget_alone_is_its_own_group():
    costs = [(2, 0), (50, 0), (2, 0), (2, 0)]
    assert _cut(costs, [(10, None)] * 4) == [[0], [1], [2, 3]]
    assert _cut([(50, 0)], [(-1, None)]) == [[0]]
    assert _cut(costs, [(-1, None)] * 4) == [[0], [1], [2], [3]]  # several ranks: groups of one


def test_device_bound_splits_groups():
    costs = [(1, 10), (1, 10), (1, 10), (1, 30), (1, 5)]
    assert _cut(costs, [(100, 25)] * 5) == [[0, 1], [2], [3], [4]]
    assert _cut(costs, [(100, None)]) == [[0, 1, 2, 3, 4]]
    assert _cut(costs, [(2, 1000)] * 3) == [[0, 1], [2, 3], [4]]


def test_file_cost_charges_getsizeof_of_the_padded_image_times_five():
    for (h, w), (win, step) in [((256, 256), (256, 164)), ((1000, 1000), (270, 80)), ((30, 300), (256, 164))]:
        padded, _ = tile._prepare_patching(np.zeros((h, w, 3), np.uint8), win, step)
        ram, dev = tile._file_cost((h, w, 3), win, step)
        assert tile._padded_shape(h, w, win, step) == padded.shape
        assert ram == sys.getsizeof(padded) * 5
        assert dev == tile.DEVICE_BYTES_PER_PX * h * w + tile.DEVICE_BYTES_PER_FILE


def test_device_charge_covers_a_mixed_group():
    """3000 PanNuke files and one 1000^2 file: the charge covers every image's own padded table (min(rows_cap,
    H*W/6 + 8) rows of 84 B), its maps and its default packed-table and point buffers, with the rest (~95 B/px) for the
    post-processing workspace."""
    shapes = [(256, 256)] * 3000 + [(1000, 1000)]
    rows_cap, pts_cap = _lib.tiles_sizes(np.array(shapes))
    tables = sum(84 * min(rows_cap, h * w // 6 + 8) for h, w in shapes)
    maps = sum((3 + 16 + 4 + 20) * h * w for h, w in shapes)
    buffers = rows_cap * 84 + pts_cap * 8
    pp = sum(95 * h * w for h, w in shapes)
    charged = sum(tile._file_cost((h, w, 3), 256, 164)[1] for h, w in shapes)
    assert tables + maps + buffers + pp <= charged
    assert tables < 3001 * 84 * 11000  # each image pays for its own size, not the largest one's (166674 rows)


def test_pack_and_split_round_trip():
    rng = np.random.default_rng(0)
    shapes = [(5, 7), (1, 1), (3, 4), (5, 7)]
    imgs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in shapes]
    packed, sh = _lib.pack_images(imgs)
    assert sh.dtype == np.int32 and sh.tolist() == [list(s) for s in shapes]
    assert np.array_equal(packed, np.concatenate([i.ravel() for i in imgs]))
    C = 4
    preds = [rng.standard_normal((h, w, C)).astype(np.float32) for h, w in shapes]
    insts = [rng.integers(0, 9, (h, w)).astype(np.int32) for h, w in shapes]
    nrows = [3, 0, 2, 1]  # image 1: an empty table
    tables = [rng.integers(0, 100, (k, 10)) for k in nrows]
    # row counts of points: image 2 has instances without contour points
    npts = [[4, 1, 3], [], [0, 0], [5]]
    pts_img = [[rng.integers(0, 50, (c, 2)).astype(np.int32) for c in rows] for rows in npts]
    ro = np.cumsum([0] + nrows).astype(np.int32)
    flat = [c for rows in npts for c in rows]
    po = np.cumsum([0] + flat).astype(np.int32)
    pts = np.concatenate([p for rows in pts_img for p in rows] or [np.zeros((0, 2), np.int32)])
    out = _lib.split_tiles(sh, np.concatenate([i.ravel() for i in insts]), np.concatenate(tables), ro,
                           np.concatenate([p.ravel() for p in preds]), pts, po)
    assert len(out) == 4
    for i, (p, im, t, offs, pt) in enumerate(out):
        assert np.array_equal(p, preds[i]) and np.array_equal(im, insts[i]) and np.array_equal(t, tables[i])
        assert len(offs) == nrows[i] + 1 and offs[0] == 0
        for r in range(nrows[i]):
            assert np.array_equal(pt[offs[r]:offs[r + 1]], pts_img[i][r])
    out = _lib.split_tiles(sh, np.concatenate([i.ravel() for i in insts]), np.concatenate(tables), ro)
    assert all(o[0] is None and o[3] is None and o[4] is None for o in out)
    assert _lib.tiles_sizes(sh) == (4 * 16, 4 * 4096)
