"""The device post-processing one stage at a time, through tests/native/libhvn_pp_probe.so (the product's own postproc.o).

a. Stage buffers of a pipeline run (size-filtered foreground, both Sobels, dist, pre-flood markers) against direct
   cv2 / scipy calls (ref_stages), bit for bit, on the shapes and contents where these kernels break; inst and the
   instance table against the C oracle.
b. Every flood kernel end to end, on maps on both sides of each size threshold of the automatic choice (the
   thresholds derived here from the kernels' shared-memory budget), read back from the profile log.
c. The flood alone (postproc_flood_only) through every kernel that fits the map, against a plain priority flood in
   this file (the referee), on constructed priorities: i.i.d. maps whose heaps spill past every shared-memory cap,
   fp32 ties, exact ties, -0.0 / +0.0, one-bucket maps, blob-size edges, W = 1 / H = 1 maps.
d. The instance table's type columns against a numpy restatement of reference post_proc.py:161-181, and the
   HVN_ERR_CAPACITY contract of hvn_postproc.
"""
import ctypes
import heapq
import os
import sys

import cv2
import numpy as np
import pytest
from scipy import ndimage

import ref_stages
from hover_net_b200 import synth

HERE = os.path.dirname(os.path.abspath(__file__))

# flood kernels (postproc.h FloodKernel) and the constants their shared-memory plan is made of (postproc.cu)
AUTO, CAL, TILE_KK, TILE, GLOBAL = 0, 1, 2, 3, 4
NAMES = {CAL: "k_watershed_cal", TILE_KK: "k_watershed_tile<true>", TILE: "k_watershed_tile<false>", GLOBAL: "k_watershed"}
BUDGET = 225 * 1024
WT_WARPS, WT_BIG, WT_SMALL_CAP, WS_CAP = 8, 2048, 256, 2048
WC_NB_BIG, WC_NB_SMALL = 2048, 256

RAN_AUTO = set()      # flood kernels seen in the profile log of a pipeline run (part b)
RAN_FORCED = set()    # flood kernels run by the flood-only entry and equal to the referee (part c)
SPILLED = set()       # (kernel, cap name) whose shared-memory heap a referee-checked flood overflowed


def _r16(b):
    return (b + 15) & ~15


def max_ids(H, W):
    return H * W // 6 + 8


def tile_cap(N, kk):
    """Entries of the large-blob heap region of k_watershed_tile for an N-px map (with / without the key table)."""
    fixed = _r16(2 * N) + (_r16(4 * N) if kk else 0) + (WT_WARPS - 1) * (WT_SMALL_CAP + 4) * 8
    cap = (BUDGET - fixed) // 8 - 4 if fixed + 64 < BUDGET else 0
    return min(cap & ~3, 16384)


def half_cap(N, kk):
    """Shared-memory entries of each of the two large-blob heaps."""
    return ((tile_cap(N, kk) + 4) // 2 - 4) & ~3


def fits(k, N):
    ids_ok = max_ids(1, N) < 32000
    if k == CAL:
        cal = _r16(8 * N) + 2 * (WC_NB_BIG * 2 + WC_NB_BIG // 8) + (WT_WARPS - 2) * (WC_NB_SMALL * 2 + WC_NB_SMALL // 8)
        return cal <= BUDGET and N < 65535 and ids_ok
    if k == TILE_KK:
        kk_room = _r16(2 * N) + _r16(4 * N) + (WT_WARPS - 1) * (WT_SMALL_CAP + 4) * 8 + (2048 + 4) * 8 <= BUDGET
        return kk_room and tile_cap(N, True) >= 1024 and N < 65536 and ids_ok
    if k == TILE:
        return tile_cap(N, False) >= 1024 and N < 65536 and ids_ok
    return k == GLOBAL


def auto_kernel(N):
    if fits(CAL, N):
        return CAL
    if fits(TILE, N):
        return TILE_KK if fits(TILE_KK, N) else TILE
    return GLOBAL


def last_n(k):
    """Largest map size (px) auto-selection floods with kernel k."""
    lo, hi = 1, 1 << 17
    assert auto_kernel(lo) <= k
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if auto_kernel(mid) <= k:
            lo = mid
        else:
            hi = mid - 1
    return lo


def test_size_thresholds_are_ordered():
    """The automatic choice moves through the four kernels in order as maps grow (no kernel is skipped)."""
    ends = [last_n(k) for k in (CAL, TILE_KK, TILE)]
    assert 0 < ends[0] < ends[1] < ends[2] == 65535
    for k, e in zip((CAL, TILE_KK, TILE), ends):
        assert auto_kernel(e) == k and auto_kernel(e + 1) == k + 1


# ------------------------------------------------------------------------------------------------ the referee
def referee(dist, mask, markers):
    """skimage's priority flood restated: mask components < 10 px are dropped, markers = markers * mask, each
    4-connected blob flooded from its marker pixels (pushed in raster order at age 0) by a heap keyed (value, age,
    raster index), neighbours up, left, right, down, the label written at push time.  Returns (inst, blobs): blobs =
    [(size, number of labels, heap high-water mark)]."""
    H, W = dist.shape
    lab, nl = ndimage.label(mask != 0)
    sizes = np.bincount(lab.ravel(), minlength=nl + 1)
    keep = (lab > 0) & (sizes >= 10)[lab]
    out = np.where(keep, markers, 0).astype(np.int32).ravel()
    d = dist.ravel().tolist()
    k = keep.ravel()
    labf = lab.ravel()
    seeds = np.flatnonzero(out > 0)
    blobs = []
    for b in np.unique(labf[seeds]):
        heap = [(d[p], 0, int(p)) for p in seeds[labf[seeds] == b]]
        nlab = len(np.unique(out[seeds[labf[seeds] == b]]))
        heapq.heapify(heap)
        hw, age = len(heap), 0
        while heap:
            _, _, p = heapq.heappop(heap)
            y, x = divmod(p, W)
            lb = out[p]
            for q in (p - W if y > 0 else -1, p - 1 if x > 0 else -1, p + 1 if x < W - 1 else -1, p + W if y < H - 1 else -1):
                if q >= 0 and k[q] and out[q] == 0:
                    age += 1
                    out[q] = lb
                    heapq.heappush(heap, (d[q], age, q))
            hw = max(hw, len(heap))
        blobs.append((int(sizes[b]), nlab, hw))
    return out.reshape(H, W), blobs


def filtered(mask):
    lab, nl = ndimage.label(mask != 0)
    return ((lab > 0) & (np.bincount(lab.ravel(), minlength=nl + 1) >= 10)[lab]).astype(np.int32)


def marker_ties(dist, mask, markers):
    """True when two marker pixels of one blob have equal priorities (where skimage's order is its heap layout)."""
    lab, _ = ndimage.label(mask != 0)
    sel = markers > 0
    pairs = set()
    for b, v in zip(lab[sel].tolist(), dist[sel].tolist()):
        if (b, v) in pairs:
            return True
        pairs.add((b, v))
    return False


# ------------------------------------------------------------------------------------------------ probe
@pytest.fixture(scope="module")
def probe():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("needs a CUDA device")
    sys.path.insert(0, os.path.join(HERE, "native"))
    try:
        import build_pp_probe
    finally:
        sys.path.pop(0)
    from hover_net_b200 import build
    build.build()
    L = ctypes.CDLL(build_pp_probe.build())
    ll, i32p = ctypes.c_longlong, ctypes.POINTER(ctypes.c_int)
    L.pp_probe_run.argtypes = [ll, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ll, ll,
                               ctypes.c_int, ll, i32p]
    L.pp_probe_buffers.argtypes = [ctypes.c_int] * 4 + [ctypes.POINTER(ctypes.c_longlong)]
    L.pp_probe_flood.argtypes = [ll, ll, ll, ctypes.c_int, ctypes.c_int, ctypes.c_int, ll, ctypes.c_int, i32p]
    L.pp_probe_max_ids.argtypes = [ctypes.c_int, ctypes.c_int]
    L.pp_probe_d2h.argtypes = [ctypes.c_void_p, ll, ll]
    yield L
    L.pp_probe_release()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run_pipeline(L, maps, nr_types=0, max_rows=None):
    """Pipeline on [n,H,W,C] maps: (inst, table, nrows, stages dict of device buffers copied to the host)."""
    import torch
    maps = np.ascontiguousarray(maps, dtype=np.float32)
    n, H, W, C = maps.shape
    mr = max_rows or max_ids(H, W)
    pred = _dev(maps)
    inst = torch.empty((n, H, W), dtype=torch.int32, device="cuda")
    table = torch.zeros((n, mr, 10), dtype=torch.int64, device="cuda")
    nrows = torch.zeros((n,), dtype=torch.int32, device="cuda")
    launches = ctypes.c_int()
    rc = L.pp_probe_run(pred.data_ptr(), n, H, W, C, nr_types, inst.data_ptr(), table.data_ptr(), mr,
                        nrows.data_ptr(), ctypes.byref(launches))
    assert rc == 0, "pp_probe_run returned %d" % rc
    ptr = (ctypes.c_longlong * 13)()
    assert L.pp_probe_buffers(n, H, W, nr_types, ptr) == 0
    st = {}
    for i, (name, dt) in enumerate([("fg", np.uint8), ("sobh", np.float64), ("sobv", np.float64),
                                    ("din", np.float64), ("dist", np.float64), ("mk0", np.uint8),
                                    ("filled", np.uint8), ("opened", np.uint8), ("L2", np.int32),
                                    ("size3", np.int32), ("id3", np.int32)]):
        buf = np.empty((n, H, W), dtype=dt)
        assert L.pp_probe_d2h(buf.ctypes.data_as(ctypes.c_void_p), ptr[i], buf.nbytes) == 0
        st[name] = buf
    # pre-flood marker labels: scipy's id of the opened component, if it kept >= 10 px; then skimage's markers * mask
    L2, size3, id3 = st["L2"].reshape(n, -1), st["size3"].reshape(n, -1), st["id3"].reshape(n, -1)
    mk = np.zeros_like(L2)
    for m in range(n):
        on = L2[m] >= 0
        r = L2[m][on]
        mk[m][on] = np.where(size3[m][r] >= 10, id3[m][r], 0)
    st["markers"] = mk.reshape(n, H, W) * st["fg"]
    return inst.cpu().numpy(), table.cpu().numpy(), nrows.cpu().numpy(), st, launches.value


# ------------------------------------------------------------------------------------------------ a. stages vs cv2/scipy
def _field(rng, H, W, sigma):
    f = cv2.GaussianBlur(rng.standard_normal((H, W)), (0, 0), sigma)
    return f / max(float(np.abs(f).max()), 1e-12)


def content_maps(H, W, seed):
    """[name, pred [H,W,3] f32] of different content for one shape."""
    rng = np.random.default_rng(seed)
    s = max(1.0, min(H, W) / 6.0)
    hv = np.stack([_field(rng, H, W, s), _field(rng, H, W, s)], -1)
    yy, xx = np.mgrid[:H, :W]
    out = []

    def add(name, npc, h=None):
        m = np.concatenate([np.asarray(npc, np.float64)[..., None], hv if h is None else h], -1)
        out.append((name, m.astype(np.float32)))

    add("smooth", 0.5 + 0.5 * _field(rng, H, W, s))
    add("const_hv", 0.5 + 0.5 * _field(rng, H, W, s), np.full((H, W, 2), 0.25))
    eps = 2.220446049250313e-16  # minmax_scale's threshold, 2^-52: a float32 exactly
    for name, r in (("range_at_eps", eps), ("range_above_eps", float(np.nextafter(np.float32(eps), np.float32(1)))),
                    ("range_below_eps", float(np.nextafter(np.float32(eps), np.float32(0))))):
        h = np.where(((yy + xx) % 3 == 0)[..., None], r, 0.0) * np.ones((1, 1, 2))
        add(name, 0.5 + 0.5 * _field(rng, H, W, s), h)
    add("np_exactly_half", np.where(_field(rng, H, W, s) > -0.2, 0.5, np.nextafter(np.float32(0.5), np.float32(0))))
    add("all_foreground", np.ones((H, W)))
    add("all_background", np.zeros((H, W)))
    # foreground on all four borders around a hole touching none of them, a notch-hole touching the top border
    ring = np.ones((H, W))
    ring[H // 3: H - H // 3, W // 3: W - W // 3] = 0.1
    ring[0: H // 4, W // 2: W // 2 + 1] = 0.1
    add("border_ring_holes", ring)
    # components of exactly 9 and 10 px (a 3x3 square and a 2x5 bar) in an empty map
    c = np.zeros((H, W))
    if H >= 3 and W >= 9:
        c[0:3, 0:3] = 0.9
        c[H - 2: H, W - 5: W] = 0.9
    elif H >= 10 or W >= 10:
        c.reshape(-1)[:9] = 0.9
        c.reshape(-1)[-10:] = 0.9
    add("sizes_9_10", c)
    if H >= 16 and W >= 16:
        out.append(("nuclei", synth.synth_pred_map(H, W, None, seed)))
    return out


SHAPES_A = ([(1, 1), (1, 7), (7, 1), (1, 64), (64, 1), (2, 2), (3, 5), (2, 300), (300, 2)]
            + [(s, s) for s in range(2, 13)] + [(20, 20), (21, 21), (22, 22), (20, 22), (22, 21)]
            + [(16, 31), (16, 32), (16, 33), (15, 64), (17, 64), (3, 1023), (3, 1025), (40, 1023), (24, 1025)]
            + [(1025, 3), (1025, 48), (2049, 2)])


def _check_stages(P, name, pm, inst, table, nrows, st, i):
    ref = ref_stages.stages(pm, P.watershed)
    assert np.array_equal(st["fg"][i], ref["blb"]), "%s: fg" % name
    assert np.array_equal(st["sobh"][i], ref["sobelh"]), "%s: sobel h" % name
    assert np.array_equal(st["sobv"][i], ref["sobelv"]), "%s: sobel v" % name
    assert np.array_equal(st["dist"][i], ref["dist"]), "%s: dist" % name
    assert np.array_equal(st["markers"][i], ref["marker"] * ref["blb"]), "%s: markers" % name
    oi, ot = P.process_table(pm, None)
    assert np.array_equal(inst[i], oi), "%s: inst (%d px differ)" % (name, int((inst[i] != oi).sum()))
    assert int(nrows[i]) == ot.shape[0] and np.array_equal(table[i, : ot.shape[0]], ot), "%s: table" % name


@pytest.mark.gpu
@pytest.mark.parametrize("hw", SHAPES_A, ids=lambda s: "%dx%d" % s)
def test_stages_equal_cv2_scipy(probe, oracle_pp, hw):
    H, W = hw
    named = content_maps(H, W, H * 7919 + W)
    maps = np.stack([m for _, m in named])
    inst, table, nrows, st, _ = run_pipeline(probe, maps)
    for i, (name, pm) in enumerate(named):
        _check_stages(oracle_pp, name, pm, inst, table, nrows, st, i)
    # every map of the batch equals its single-map run
    for i, (name, pm) in enumerate(named):
        i1, t1, n1, s1, _ = run_pipeline(probe, pm[None])
        assert np.array_equal(i1[0], inst[i]) and int(n1[0]) == int(nrows[i]), name
        assert np.array_equal(t1[0, : n1[0]], table[i, : nrows[i]]), name
        for k in ("fg", "sobh", "sobv", "dist", "markers"):
            assert np.array_equal(s1[k][0], st[k][i]), "%s: %s differs between batch and single map" % (name, k)


TINY_THIN = [hw for hw in SHAPES_A if min(hw) <= 12 or max(hw) >= 1023]


@pytest.mark.parametrize("hw", TINY_THIN, ids=lambda s: "%dx%d" % s)
def test_oracle_stages_pinned_on_tiny_and_thin_maps(oracle_pp, hw):
    """CPU: the C oracle, stage by stage, equals cv2 / scipy on the maps smaller than the Sobel radius or one pixel
    thick, so that it can referee the device there."""
    H, W = hw
    for name, pm in content_maps(H, W, H * 7919 + W):
        inst, st = oracle_pp.proc_np_hv(pm, True)
        ref = ref_stages.stages(pm, oracle_pp.watershed)
        for k in st:
            assert np.array_equal(st[k], ref[k]), "%s: %s" % (name, k)
        assert np.array_equal(inst, ref["inst"]), name


@pytest.mark.gpu
def test_many_ids_tall_map(probe, oracle_pp):
    """> 1024 marker ids over > 2048 rows: the carry of k_row_scan and k_table_rows' blocks of 1024 ids."""
    pm = synth.synth_pred_map(2049, 192, None, 4, density=1.0 / 120.0)
    inst, table, nrows, st, _ = run_pipeline(probe, pm[None])
    assert int(st["id3"].max()) > 1024 and int(nrows[0]) > 1024
    _check_stages(oracle_pp, "tall", pm, inst, table, nrows, st, 0)


# ------------------------------------------------------------------------------------------------ b. floods by size
def _threshold_shapes():
    shapes = [(164, 164), (165, 165), (166, 166), (182, 182), (183, 183), (255, 257), (256, 256)]
    for k in (CAL, TILE_KK, TILE):
        e = last_n(k)
        h = int(np.sqrt(e))
        shapes += [(h, e // h), (h, e // h + 1)]
    return sorted(set(shapes))


def _flood_maps(H, W):
    rng = np.random.default_rng(H * 131 + W)
    maps = []
    for s in range(2):  # CNN-like smooth fields: large irregular blobs with several markers each
        m = np.stack([cv2.GaussianBlur(rng.standard_normal((H, W)), (0, 0), g) for g in (6, 4, 4)], -1)
        m = m / np.abs(m).max((0, 1))
        m[..., 0] = 0.55 + 0.5 * m[..., 0]
        maps.append(m.astype(np.float32))
    maps.append(synth.synth_pred_map(H, W, None, 1, density=1.0 / 350.0))  # crowded: touching nuclei
    return np.stack(maps)


def _multi_marker_blobs(P, pm):
    """(size, labels) of every foreground blob the oracle floods with >= 2 marker labels."""
    _, st = P.proc_np_hv(pm, True)
    lab, _ = ndimage.label(st["blb"])
    mk = st["marker"] * st["blb"]
    out = []
    for b in np.unique(lab[mk > 0]):
        sel = lab == b
        n = len(np.unique(mk[sel & (mk > 0)]))
        if n >= 2:
            out.append((int(sel.sum()), n))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("hw", _threshold_shapes(), ids=lambda s: "%dx%d" % s)
def test_flood_kernel_by_size(oracle_pp, hw):
    from hover_net_b200 import _lib
    H, W = hw
    maps = _flood_maps(H, W)
    blobs = sum((_multi_marker_blobs(oracle_pp, m) for m in maps), [])
    assert any(s >= WT_BIG for s, _ in blobs) and any(s < WT_BIG for s, _ in blobs), "both warp passes must run"
    c = _lib.Context(0)
    try:
        c.set_option("profile", 3)
        inst, table, nrows = c.postproc(maps, None)
        ran = [NAMES[k] for k in NAMES if any(l.split()[1:2] == [NAMES[k]] for l in c.debug_log().split("\n")
                                              if l.startswith("pp "))]
    finally:
        c.close()
    assert ran == [NAMES[auto_kernel(H * W)]], ran
    RAN_AUTO.add(auto_kernel(H * W))
    for i in range(maps.shape[0]):
        oi, ot = oracle_pp.process_table(maps[i], None)
        assert np.array_equal(inst[i], oi), "map %d: %d px differ" % (i, int((inst[i] != oi).sum()))
        assert int(nrows[i]) == ot.shape[0] and np.array_equal(table[i, : ot.shape[0]], ot)


# ------------------------------------------------------------------------------------------------ c. the flood alone
def _blob_mask(H, W, y0, x0, h, w):
    m = np.zeros((H, W), np.uint8)
    m[y0: y0 + h, x0: x0 + w] = 1
    return m


def _seed(rng, mask, k, first=1):
    """k marker pixels with labels first.. at random positions of the mask."""
    mk = np.zeros(mask.shape, np.int32)
    pix = np.flatnonzero(mask.ravel())
    sel = rng.choice(pix, size=min(k, pix.size), replace=False)
    mk.ravel()[sel] = np.arange(first, first + sel.size)
    return mk


def flood_cases():
    """name -> (dist [n,H,W] f64, mask u8, markers i32)."""
    rng = np.random.default_rng(2024)
    cases = {}

    def one(name, d, m, k):
        cases[name] = (d[None], m[None], k[None])

    # i.i.d. uniform priorities over one blob with a few markers: the heap grows past every shared-memory cap
    m = _blob_mask(64, 64, 7, 9, 40, 50)  # 2000 px: a small blob (< WT_BIG)
    one("iid_small_blob", rng.uniform(size=(64, 64)), m, _seed(rng, m, 5))
    for H, W in ((120, 120), (181, 181), (200, 200), (255, 257), (256, 256)):
        m = _blob_mask(H, W, 0, 0, H, W)
        one("iid_%dx%d" % (H, W), rng.uniform(size=(H, W)), m, _seed(rng, m, 6))
    # priorities that tie in fp32 but differ in fp64 (fp32 values plus 0-2 ulps), and fp32 values quantised to 8 levels
    base = rng.integers(0, 8, size=(96, 96)).astype(np.float32).astype(np.float64) / 8.0
    d = base.copy()
    ulps = rng.integers(0, 3, size=d.shape)
    for u in (1, 2):
        sel = ulps >= u
        d[sel] = np.nextafter(d[sel], np.inf)
    m = np.ones((96, 96), np.uint8)
    one("fp32_ties_fp64_differs", d, m, _seed(rng, m, 12))
    # equal non-marker priorities (age order), -0.0 / +0.0, everything equal (calendar scale 0: one bucket)
    d = np.full((80, 80), 0.25)
    k = _seed(rng, np.ones((80, 80), np.uint8), 9)
    d[k > 0] = rng.uniform(size=int((k > 0).sum())) - 1.0
    one("equal_priorities", d, np.ones((80, 80), np.uint8), k)
    d = np.where(rng.uniform(size=(80, 80)) < 0.5, -0.0, 0.0)
    d[k > 0] = rng.uniform(size=int((k > 0).sum())) - 1.0
    one("signed_zeros", d, np.ones((80, 80), np.uint8), k)
    one("all_equal", np.full((80, 80), -0.5), np.ones((80, 80), np.uint8), _seed(rng, np.ones((80, 80), np.uint8), 7))
    # clustered in a tiny range with a few far outliers: nearly everything in one calendar bucket
    d = 0.3 + rng.uniform(size=(100, 100)) * 1e-9
    d.ravel()[rng.choice(10000, 5, replace=False)] = [-50.0, 40.0, 1e6, -1e6, 7.0]
    one("clustered_outliers", d, np.ones((100, 100), np.uint8), _seed(rng, np.ones((100, 100), np.uint8), 10))
    # blobs of 2047 and 2048 px (WT_BIG), 10 px, a one-pixel-wide snake, blobs on every border
    H, W = 140, 150
    m = np.zeros((H, W), np.uint8)
    m[0:23, 0:89] = 1; m[0, 89] = 1                       # 2048 px, touches top and left
    m[H - 23: H, W - 89: W] = 1; m[H - 1, W - 89] = 0      # 2047 px with the next line, touches bottom and right
    m[H - 24, W - 1] = 1
    m[60:62, 70:75] = 1                                   # 10 px
    m[30:110:2, 20:60] = 1; m[31:110:4, 59] = 1; m[33:110:4, 20] = 1  # snake
    m[40:100, W - 1] = 1; m[40:100, W - 3] = 1; m[40, W - 3: W] = 1   # on the right border
    d = rng.uniform(size=(H, W))
    one("blob_size_edges", d, m, _seed(rng, m, 40))
    # hundreds of labels in one blob, up to the pipeline's id bound N/6 + 8
    H, W = 90, 110
    m = np.ones((H, W), np.uint8)
    k = _seed(rng, m, max_ids(H, W) - 1)
    one("many_labels", rng.uniform(size=(H, W)), m, k)
    # several maps per call with different blob counts (per-map heap arenas)
    ds, ms, ks = [], [], []
    for nb in (1, 4, 12, 0, 30):
        d = rng.uniform(size=(120, 128))
        m = np.zeros((120, 128), np.uint8)
        for b in range(nb):
            y, x = (b // 6) * 24, (b % 6) * 21
            m[y: y + 20 + (b % 3), x: x + 18] = 1
        if nb == 1:
            m[:] = 1
        ds.append(d); ms.append(m); ks.append(_seed(rng, m, 3 * nb + 2))
    cases["maps_with_different_blob_counts"] = (np.stack(ds), np.stack(ms), np.stack(ks))
    # W = 1 and H = 1 maps: blobs ending at the last pixel, and not
    for H, W in ((37, 1), (300, 1), (1, 37), (1, 300)):
        m = np.ones((H, W), np.uint8)
        m.ravel()[15] = 0
        one("thin_%dx%d" % (H, W), rng.uniform(size=(H, W)), m, _seed(rng, m, 4))
    m = np.ones((64, 1), np.uint8)
    m[-1] = 0
    one("thin_64x1_last_px_off", rng.uniform(size=(64, 1)), m, _seed(rng, m, 3))
    # exact ties between age-0 marker pixels (raster order decides; the oracle differs there by design)
    d = np.round(rng.uniform(size=(60, 60)) * 4) / 4
    m = np.ones((60, 60), np.uint8)
    k = _seed(rng, m, 80)
    d[k > 0] = 0.5
    one("marker_ties", d, m, k)
    return cases


CASES = flood_cases()


def run_flood(L, d, m, k, choice):
    import torch
    n, H, W = d.shape
    dd, mm, kk = _dev(d.astype(np.float64)), _dev(m.astype(np.uint8)), _dev(k.astype(np.int32))
    inst = torch.full((n, H, W), -7, dtype=torch.int32, device="cuda")
    kern = ctypes.c_int(-1)
    rc = L.pp_probe_flood(dd.data_ptr(), mm.data_ptr(), kk.data_ptr(), n, H, W, inst.data_ptr(), choice,
                          ctypes.byref(kern))
    return rc, kern.value, inst.cpu().numpy()


def test_referee_equals_oracle_watershed(oracle_pp):
    """On maps without tied marker pixels the referee is skimage's flood as the oracle restates it."""
    for name, (d, m, k) in CASES.items():
        for i in range(d.shape[0]):
            if marker_ties(d[i], filtered(m[i]), k[i]) or d.shape[1] * d.shape[2] > 40000:
                continue
            f = filtered(m[i])
            ref, _ = referee(d[i], m[i], k[i])
            assert np.array_equal(ref, oracle_pp.watershed(d[i], k[i] * f, f)), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_flood_only_every_kernel_equals_referee(probe, name):
    d, m, k = CASES[name]
    n, H, W = d.shape
    assert int(k.max()) < max_ids(H, W)
    refs = [referee(d[i], m[i], k[i]) for i in range(n)]
    ran = []
    for choice in (AUTO, CAL, TILE_KK, TILE, GLOBAL):
        rc, kern, inst = run_flood(probe, d, m, k, choice)
        if choice != AUTO and not fits(choice, H * W):
            assert rc == -1, "%s: a forced kernel that does not fit must be refused, not run" % NAMES[choice]
            continue
        assert rc == 0, "%s: rc %d" % (name, rc)
        assert kern == (auto_kernel(H * W) if choice == AUTO else choice)
        for i in range(n):
            bad = int((inst[i] != refs[i][0]).sum())
            assert bad == 0, "%s map %d, %s: %d px differ from the referee" % (name, i, NAMES[kern], bad)
        ran.append(kern)
        RAN_FORCED.add(kern)
        for size, nlab, hw in (b for r in refs for b in r[1]):
            if nlab < 2:
                continue  # single-label blobs are filled without a flood
            if kern in (TILE_KK, TILE):
                if size < WT_BIG and hw > WT_SMALL_CAP:
                    SPILLED.add((kern, "WT_SMALL_CAP"))
                if size >= WT_BIG and hw > half_cap(H * W, kern == TILE_KK):
                    SPILLED.add((kern, "half_cap"))
            if kern == GLOBAL and hw > WS_CAP:
                SPILLED.add((kern, "WS_CAP"))
    assert GLOBAL in ran


# ------------------------------------------------------------------------------------------------ d. instance table
def type_rows(inst, tp, ids, valid_range=None):
    """post_proc.py:161-181 restated: (type, type_cnt, type_prob) per id; tp truncated like astype(int32).  With
    valid_range = nr_types only values in [0, nr_types) are counted (the device's k_table_accum)."""
    t = tp.astype(np.int32)
    out = []
    for i in ids:
        sel = inst == i
        v = t[sel]
        if valid_range is not None:
            v = v[(v >= 0) & (v < valid_range)]
        if v.size == 0:
            out.append((-1, 0, 0.0))
            continue
        tl, tc = np.unique(v, return_counts=True)
        lst = sorted(zip(tl.tolist(), tc.tolist()), key=lambda x: x[1], reverse=True)
        typ = lst[0][0]
        if typ == 0 and len(lst) > 1:
            typ = lst[1][0]
        cnt = dict(lst)[typ]
        out.append((typ, cnt, float(cnt / (sel.sum() + 1.0e-6))))
    return out


def _typed_map(P, nt):
    pm = synth.synth_pred_map(164, 164, nt, 2)
    inst, _ = P.process_table(pm, nt)
    rng = np.random.default_rng(7)
    tp = np.zeros(inst.shape, np.float32)
    ids = [i for i in np.unique(inst) if i > 0]
    for j, i in enumerate(ids):
        ys, xs = np.nonzero(inst == i)
        n = ys.size
        o = rng.permutation(n)
        v = np.zeros(n, np.float32)
        case = j % 5
        if case == 0:    # tie between non-zero types 3 and 2 (the smaller wins), one or two px of type 1
            q = (n - 1) // 2
            v[o[:q]], v[o[q: 2 * q]], v[o[2 * q:]] = 3, 2, 1
        elif case == 1:  # type 0 wins, runner-up tied between 4 and 5
            q = n // 4
            v[o[:q]], v[o[q: 2 * q]], v[o[2 * q:]] = 5, 4, 0
        elif case == 2:  # type 0 only
            pass
        elif case == 3:  # negative fractions truncate to 0; 2.9 truncates to 2
            v[o[: n // 2]] = -0.75
            v[o[n // 2:]] = 2.9
        else:            # mixture with values past nr_types and below 0 (ignored on the device)
            v[o[: n // 2]] = nt + 1
            v[o[n // 2: 3 * n // 4]] = -1.5
            v[o[3 * n // 4:]] = 1
        tp[ys, xs] = v
    pm[..., 0] = tp
    return pm, ids


@pytest.mark.gpu
def test_instance_table_types(probe, oracle_pp):
    from hover_net_b200.models.hovernet.post_proc import process
    nt = 6
    pm, ids = _typed_map(oracle_pp, nt)
    inst, table, nrows, _, _ = run_pipeline(probe, pm[None], nr_types=nt)
    rows = table[0, : nrows[0]]
    assert rows[:, 0].tolist() == ids
    want = type_rows(inst[0], pm[..., 0], ids, valid_range=nt)
    assert [(int(r[8]), int(r[9])) for r in rows] == [(w[0], w[1]) for w in want]
    full = type_rows(inst[0], pm[..., 0], ids)
    # the deliberate deviation: values outside [0, nr_types) are counted by the reference, ignored here
    dev = [j for j in range(len(ids)) if j % 5 == 4]
    assert dev and all(full[j][0] != want[j][0] for j in dev)
    assert all(full[j] == want[j] for j in range(len(ids)) if j % 5 != 4)
    _, info = process(pm, nr_types=nt)
    for j, i in enumerate(ids):
        if i in info:
            assert info[i]["type"] == want[j][0] and info[i]["type_prob"] == want[j][2]


@pytest.mark.gpu
def test_capacity_error_and_retry():
    from hover_net_b200 import _lib
    maps = np.stack([synth.synth_pred_map(164, 164, 6, s) for s in range(3)])
    c = _lib.Context(0)
    try:
        inst, table, nrows = c.postproc(maps, 6, max_rows=max_ids(164, 164))
        need = int(nrows.max())
        assert need > 4
        p = np.ascontiguousarray(maps)
        small = need - 3
        inst2 = np.empty(inst.shape, np.int32)
        table2 = np.zeros((3, small, 10), np.int64)
        nrows2 = np.zeros(3, np.int32)
        rc = _lib.lib().hvn_postproc(c._h, _lib._ptr(p), 3, 164, 164, 4, 6, _lib._ptr(inst2), _lib._ptr(table2), small,
                                     _lib._ptr(nrows2))
        assert rc == -4 and np.array_equal(nrows2, nrows)
        retry = c.postproc(maps, 6, max_rows=small)
        assert np.array_equal(retry[0], inst) and np.array_equal(retry[2], nrows)
        assert np.array_equal(retry[1], table[:, : retry[1].shape[1]])
    finally:
        c.close()


# ------------------------------------------------------------------------------------------------ coverage
@pytest.mark.gpu
def test_zz_every_flood_kernel_ran_and_every_cap_spilled():
    """Runs last in this module: the four flood kernels ran both by automatic choice and forced, equal to their
    referees, and every shared-memory heap cap was exceeded by at least one referee-checked flood."""
    assert RAN_AUTO == {CAL, TILE_KK, TILE, GLOBAL}, RAN_AUTO
    assert RAN_FORCED == {CAL, TILE_KK, TILE, GLOBAL}, RAN_FORCED
    want = {(TILE_KK, "WT_SMALL_CAP"), (TILE_KK, "half_cap"), (TILE, "WT_SMALL_CAP"), (TILE, "half_cap"),
            (GLOBAL, "WS_CAP")}
    assert want <= SPILLED, sorted(want - SPILLED)
