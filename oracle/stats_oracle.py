"""CPU restatement of the instance pair table (hvn_inst_pairs), numpy only: np.unique over the combined (t, p)
keys of every pixel with t > 0 or p > 0, with return_counts.  Same interface as
hover_net_b200.metrics.stats_utils.pair_table: rows [k,3] int64 (t, p, count) sorted by (t, p) within each map,
offs [n+1] int64."""
import numpy as np


def pair_table(true, pred=None):
    t = np.asarray(true, dtype=np.int64)
    p = np.zeros_like(t) if pred is None else np.asarray(pred, dtype=np.int64)
    if t.ndim == 2:
        t, p = t[None], p[None]
    if t.shape != p.shape:
        raise ValueError("shapes differ")
    if (t < 0).any() or (p < 0).any():
        raise ValueError("negative instance id")
    rows, offs = [], [0]
    for m in range(t.shape[0]):
        key = (t[m] << 32) | p[m]
        key = key[key > 0]
        u, c = np.unique(key, return_counts=True)
        rows.append(np.stack([u >> 32, u & 0xFFFFFFFF, c.astype(np.int64)], axis=1))
        offs.append(offs[-1] + u.size)
    return np.concatenate(rows, axis=0).reshape(-1, 3), np.array(offs, dtype=np.int64)
