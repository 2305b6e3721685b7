"""GPU checks of the instance metrics: the device pair table (hvn_inst_pairs*) equals the numpy oracle, and the
metrics mirror reproduces every golden reference outcome bit-exactly with the device table."""
import numpy as np
import pytest

from hover_net_b200 import synth
from oracle import stats_oracle as O

import stats_golden as G

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from hover_net_b200.models.hovernet.post_proc import _ctx
    return _ctx()  # post-processing-only context, the one the metrics use


def _same_table(ctx, true, pred, **kw):
    rows, offs = ctx.inst_pairs(true, pred, **kw)
    orows, ooffs = O.pair_table(true, pred)
    assert np.array_equal(offs, ooffs)
    assert np.array_equal(rows, orows)
    return rows


def test_stats_utils_matches_reference():
    from hover_net_b200.metrics import stats_utils
    G.check_stats_utils(stats_utils)


def test_compute_stats_matches_reference(tmp_path, capsys):
    from hover_net_b200 import compute_stats
    G.check_compute_stats(compute_stats, tmp_path, capsys)


def test_batched_and_single(ctx):
    g = G.load("stats_utils.npz")
    t = np.stack([g["true_%d" % k] for k in range(8)])
    p = np.stack([g["pred_%d" % k] for k in range(8)])
    _same_table(ctx, t, p)
    for k in range(8):
        _same_table(ctx, t[k], p[k])
    _same_table(ctx, t, None)
    _same_table(ctx, t[3], None)


def test_large_map():
    """4096^2 with ~18k instances, prediction shifted and relabelled."""
    from hover_net_b200.models.hovernet.post_proc import _ctx
    t = synth.tiled_instances(4096, 4096, seed=1)
    assert t.max() > 15000
    p = np.roll(t, (3, -2), (0, 1))
    p = np.where(p > 0, p + 7, 0).astype(np.int32)
    rows = _same_table(_ctx(), t, p)
    assert rows[:, 2].sum() == int(((t > 0) | (p > 0)).sum())


def test_random_ids_capacity_retry(ctx):
    """pairs ~ pixels: full hash tables, and a too-small cap answered by HVN_ERR_CAPACITY + retry."""
    rng = np.random.default_rng(3)
    t = rng.integers(0, 1 << 20, (2, 700, 530)).astype(np.int32)
    p = rng.integers(0, 1 << 20, (2, 700, 530)).astype(np.int32)
    rows = _same_table(ctx, t, p, cap=16)
    assert rows.shape[0] > 0.99 * t.size
    # device variant: too small a cap reports the size and writes nothing
    n, H, W = t.shape
    d_t, d_p = ctx.malloc(t.nbytes), ctx.malloc(p.nbytes)
    d_offs, d_rows = ctx.malloc(8 * (n + 1)), ctx.malloc(24 * 16)
    try:
        ctx.h2d(d_t, t, t.nbytes)
        ctx.h2d(d_p, p, p.nbytes)
        assert ctx.inst_pairs_dev(d_t, d_p, n, H, W, d_rows, 16, d_offs) is False
        offs = np.zeros(n + 1, np.int64)
        ctx.d2h(offs, d_offs, offs.nbytes)
        ctx.sync()
        assert np.array_equal(offs, O.pair_table(t, p)[1])
    finally:
        for d in (d_t, d_p, d_offs, d_rows):
            ctx.free(d)


def test_one_instance_everywhere(ctx):
    """Maximum contention: every pixel adds to one key; the count must be exactly H*W."""
    t = np.ones((2048, 2048), np.int32)
    rows, offs = ctx.inst_pairs(t, t)
    assert rows.tolist() == [[1, 1, 2048 * 2048]]
    rows, offs = ctx.inst_pairs(t, None)
    assert rows.tolist() == [[1, 0, 2048 * 2048]]


def test_ids_near_int32_max(ctx):
    rng = np.random.default_rng(8)
    base = synth.synth_instances(300, 300, seed=4)
    t = np.where(base > 0, np.int64(2 ** 31 - 1) - base, 0).astype(np.int32)
    p = np.where(np.roll(base, 5, 1) > 0, np.int64(2 ** 31 - 1) - rng.permutation(400)[np.roll(base, 5, 1)], 0)
    rows = _same_table(ctx, t, p.astype(np.int32))
    assert rows[:, 0].max() == 2 ** 31 - 2


def test_negative_id_is_invalid(ctx):
    from hover_net_b200 import _lib
    t = np.zeros((40, 50), np.int32)
    t[10, 20] = -3
    with pytest.raises(_lib.HvnError) as e:
        ctx.inst_pairs(t, None)
    assert e.value.code == -1
    with pytest.raises(_lib.HvnError) as e:
        ctx.inst_pairs(np.zeros_like(t), t)
    assert e.value.code == -1


def test_device_resident_postproc_output(ctx):
    """hvn_postproc_dev output fed straight into hvn_inst_pairs_dev gives the host path's table."""
    n, H, W = 4, 164, 164
    pm = np.stack([synth.synth_pred_map(H, W, None, s) for s in range(n)])
    true = np.stack([synth.synth_instances(H, W, seed=s) for s in range(n)])
    max_rows, cap = 1024, 1 << 16
    bufs = [ctx.malloc(b) for b in (pm.nbytes, 4 * n * H * W, 80 * n * max_rows, 4 * n, true.nbytes, 24 * cap,
                                    8 * (n + 1))]
    d_pm, d_inst, d_tab, d_nr, d_true, d_rows, d_offs = bufs
    try:
        ctx.h2d(d_pm, pm, pm.nbytes)
        ctx.h2d(d_true, true, true.nbytes)
        ctx.postproc_dev(d_pm, n, H, W, 3, None, d_inst, d_tab, max_rows, d_nr)
        assert ctx.inst_pairs_dev(d_true, d_inst, n, H, W, d_rows, cap, d_offs)
        offs = np.zeros(n + 1, np.int64)
        ctx.d2h(offs, d_offs, offs.nbytes)
        ctx.sync()
        rows = np.zeros((int(offs[-1]), 3), np.int64)
        ctx.d2h(rows, d_rows, rows.nbytes)
        inst = np.zeros((n, H, W), np.int32)
        ctx.d2h(inst, d_inst, inst.nbytes)
        ctx.sync()
    finally:
        for d in bufs:
            ctx.free(d)
    m = np.repeat(np.arange(n), np.diff(offs))
    rows = rows[np.lexsort((rows[:, 1], rows[:, 0], m))]
    hrows, hoffs = ctx.inst_pairs(true, inst)
    assert inst.max() > 0
    assert np.array_equal(offs, hoffs) and np.array_equal(rows, hrows)
