"""CPU checks of the instance metrics: the numpy pair-table oracle against the golden maps, and the metrics'
host finishing code, fed the oracle's table instead of the device's, against every golden reference outcome."""
import numpy as np
import pytest

from oracle import stats_oracle as O

import stats_golden as G


@pytest.fixture
def oracle_tables(monkeypatch):
    from hover_net_b200 import compute_stats
    from hover_net_b200.metrics import stats_utils
    monkeypatch.setattr(stats_utils, "pair_table", O.pair_table)
    return stats_utils, compute_stats


def _brute(true, pred):
    """Intersections and areas straight from the masks (what the reference computes)."""
    out = {}
    for t in np.unique(true):
        for p in np.unique(pred[true == t]):
            if t or p:
                out[(int(t), int(p))] = int(((true == t) & (pred == p)).sum())
    return out


def test_oracle_table_matches_masks():
    g = G.load("stats_utils.npz")
    for k in range(9):  # the synthetic and tie cases
        true, pred = g["true_%d" % k], g["pred_%d" % k]
        rows, offs = O.pair_table(true, pred)
        assert list(offs) == [0, rows.shape[0]]
        assert {(int(t), int(p)): int(c) for t, p, c in rows} == _brute(true, pred)
        order = np.lexsort((rows[:, 1], rows[:, 0]))
        assert np.array_equal(order, np.arange(rows.shape[0]))
        # areas are row / column sums
        ids, areas = np.unique(true[true > 0], return_counts=True)
        tr = rows[rows[:, 0] > 0]
        assert np.array_equal(np.unique(tr[:, 0]), ids)
        assert np.array_equal(np.array([tr[tr[:, 0] == i, 2].sum() for i in ids]), areas)


def test_oracle_batched_and_null_pred():
    g = G.load("stats_utils.npz")
    t = np.stack([g["true_%d" % k] for k in range(3)])
    p = np.stack([g["pred_%d" % k] for k in range(3)])
    rows, offs = O.pair_table(t, p)
    for k in range(3):
        r1, _ = O.pair_table(t[k], p[k])
        assert np.array_equal(rows[offs[k]:offs[k + 1]], r1)
    rows, offs = O.pair_table(t[0])
    ids, areas = np.unique(t[0][t[0] > 0], return_counts=True)
    assert np.array_equal(rows, np.stack([ids, 0 * ids, areas], 1))


def test_stats_utils_matches_reference(oracle_tables):
    G.check_stats_utils(oracle_tables[0])


def test_compute_stats_matches_reference(oracle_tables, tmp_path, capsys):
    G.check_compute_stats(oracle_tables[1], tmp_path, capsys)


def test_cli_parses_reference_options(oracle_tables, tmp_path, capsys):
    C = oracle_tables[1]
    C.main(["--mode", "instance", "--pred_dir", str(tmp_path), "--true_dir", str(tmp_path)])
    assert capsys.readouterr().out.split("\n")[0] == str(tmp_path)
