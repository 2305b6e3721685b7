"""Drop-in for reference `metrics/stats_utils.py`: the nuclei instance-segmentation metrics.

Every metric needs one thing per pixel: the contingency table of (true id, pred id) pairs with their pixel counts.
`pair_table` computes it on the device in one pass over both maps (csrc/stats.cu, `hvn_inst_pairs`); the rest is
host work on a few thousand integers.  The reference instead builds a full-map mask per instance and per
overlapping pair, O(instances * pixels).

Results are bit-identical to the reference: every quantity it sums is an integer count (exact here as well), and
its floating-point steps are reproduced on the same values in the same order -- `inter / (union + 1e-6)` for the
AJI argmax (ties go to the smallest pred id), `inter / (total - inter)` for PQ, and the PQ `paired_iou` array in
row-major (true id, pred id) order, because numpy's pairwise sum depends on the order.  The Munkres steps (AJI+,
and PQ with `match_iou < 0.5`) call `scipy.optimize.linear_sum_assignment` on the same dense N_true x N_pred
float64 IoU matrix the reference builds, zeros included, so they need that much host memory, as the reference does:
which optimal assignment scipy picks among ties decides the AJI+ value.

One deliberate difference: the `get_fast_*` functions require instance ids that are exactly {0, 1, ..., N} (call
`remap_label` first, as the reference's docstrings say) and raise IndexError otherwise.  The reference raises
IndexError in most such cases too, but in some (e.g. pred ids {1, 3, 4}) it silently scores the wrong masks.
"""
import numpy as np
from scipy.optimize import linear_sum_assignment
from scipy.spatial.distance import cdist

from ..models.hovernet.post_proc import _ctx


def pair_table(true, pred):
    """(rows [k,3] int64 (t, p, count) sorted by (t, p) within each map, offs [n+1]) of maps [H,W] or [n,H,W];
    pred None means an all-zero map.  The only pixel work of this module; it runs on the device."""
    return _ctx().inst_pairs(true, pred)


class _Pairs:
    """The pair table of one map pair and what the metrics read from it."""

    def __init__(self, rows, npx):
        self.t, self.p, self.c = (np.ascontiguousarray(rows[:, k]) for k in range(3))
        bg = npx - int(self.c.sum())  # pixels where both ids are 0
        self.t_has0 = bool(bg > 0 or (self.t == 0).any())
        self.p_has0 = bool(bg > 0 or (self.p == 0).any())
        tm, pm = self.t > 0, self.p > 0
        self.tid, first = np.unique(self.t[tm], return_index=True)  # rows are sorted by t
        self.tarea = np.add.reduceat(self.c[tm], first) if first.size else np.zeros(0, np.int64)
        self.pid, inv = np.unique(self.p[pm], return_inverse=True)
        self.parea = np.zeros(self.pid.size, np.int64)
        np.add.at(self.parea, inv, self.c[pm])
        both = tm & pm  # the overlaps, in row-major (t, p) order
        self.it, self.ip, self.inter = self.t[both], self.p[both], self.c[both]

    def renamed(self):
        """The table of the maps after remap_label(by_size=False): ids become their rank (an order-preserving
        bijection, so the (t, p) order is kept)."""
        out = object.__new__(_Pairs)
        out.__dict__.update(self.__dict__)
        out.t = np.where(self.t > 0, np.searchsorted(self.tid, self.t) + 1, 0)
        out.p = np.where(self.p > 0, np.searchsorted(self.pid, self.p) + 1, 0)
        out.it = np.searchsorted(self.tid, self.it) + 1
        out.ip = np.searchsorted(self.pid, self.ip) + 1
        out.tid = np.arange(1, self.tid.size + 1, dtype=self.tid.dtype)
        out.pid = np.arange(1, self.pid.size + 1, dtype=self.pid.dtype)
        return out

    def check_contiguous(self):
        for has0, ids, name in ((self.t_has0, self.tid, "true"), (self.p_has0, self.pid, "pred")):
            if not has0 or (ids.size and ids[-1] != ids.size):
                raise IndexError("%s instance ids are not contiguous {0, 1, ..., N}: call remap_label first" % name)

    def areas(self):
        """Areas of the true / pred instance of every overlap (ids are contiguous)."""
        return self.tarea[self.it - 1], self.parea[self.ip - 1]


def _table(true, pred=None):
    true = np.asarray(true)
    rows, _ = pair_table(true, pred)
    return _Pairs(rows, true.size)


def _ids(tab, which, dtype):
    n = tab.tid.size if which == "t" else tab.pid.size
    return np.arange(1, n + 1, dtype=dtype)


def _unpaired_area(ids_area, paired_idx):
    keep = np.ones(ids_area.size, bool)
    keep[np.asarray(paired_idx, dtype=np.int64)] = False
    return int(ids_area[keep].sum())


def _aji_iou(tab):
    ta, pa = tab.areas()
    union = ta + pa - tab.inter
    return tab.inter.astype(np.float64) / (union.astype(np.float64) + 1.0e-6), union


def _dense(tab, vals):
    m = np.zeros((tab.tid.size, tab.pid.size), dtype=np.float64)
    m[tab.it - 1, tab.ip - 1] = vals
    return m


def _aji(tab):
    tab.check_contiguous()
    if tab.pid.size == 0:
        raise ValueError("attempt to get argmax of an empty sequence")
    iou, union = _aji_iou(tab)
    # argmax over each true row: the largest IoU, ties to the smallest pred id (all overlaps have IoU > 0)
    order = np.lexsort((tab.ip, -iou, tab.it))
    first = np.ones(order.size, bool)
    first[1:] = tab.it[order][1:] != tab.it[order][:-1]
    sel = order[first]
    inter = int(tab.inter[sel].sum())
    un = int(union[sel].sum())
    un += _unpaired_area(tab.tarea, tab.it[sel] - 1) + _unpaired_area(tab.parea, tab.ip[sel] - 1)
    return np.float64(inter) / np.float64(un)


def _aji_plus(tab):
    tab.check_contiguous()
    iou, union = _aji_iou(tab)
    rt, rp = linear_sum_assignment(-_dense(tab, iou))
    pos = np.searchsorted(tab.it * (tab.pid.size + 1) + tab.ip, (rt + 1) * (tab.pid.size + 1) + (rp + 1))
    hit = pos < tab.it.size
    hit[hit] = (tab.it[pos[hit]] == rt[hit] + 1) & (tab.ip[pos[hit]] == rp[hit] + 1)  # assigned pairs that overlap
    inter = int(tab.inter[pos[hit]].sum())
    un = int(union[pos[hit]].sum())
    un += _unpaired_area(tab.tarea, rt[hit]) + _unpaired_area(tab.parea, rp[hit])
    return np.float64(inter) / np.float64(un)


def _pq(tab, match_iou, id_dtype):
    tab.check_contiguous()
    ta, pa = tab.areas()
    iou = tab.inter.astype(np.float64) / (ta + pa - tab.inter).astype(np.float64)
    if match_iou >= 0.5:  # every IoU > 0.5 pairing is unique: no assignment needed
        sel = iou > match_iou
        paired_true = tab.it[sel].astype(np.intp)
        paired_pred = tab.ip[sel].astype(np.intp)
        paired_iou = iou[sel]
    else:
        dense = _dense(tab, iou)
        rt, rp = linear_sum_assignment(-dense)
        piou = dense[rt, rp]
        keep = piou > match_iou
        paired_true = list(rt[keep] + 1)
        paired_pred = list(rp[keep] + 1)
        paired_iou = piou[keep]
    tid, pid = _ids(tab, "t", id_dtype[0]), _ids(tab, "p", id_dtype[1])
    unpaired_true = list(tid[~np.isin(tid, np.asarray(paired_true, dtype=np.int64))])
    unpaired_pred = list(pid[~np.isin(pid, np.asarray(paired_pred, dtype=np.int64))])
    tp, fp, fn = len(paired_true), len(unpaired_pred), len(unpaired_true)
    dq = tp / (tp + 0.5 * fp + 0.5 * fn)
    sq = paired_iou.sum() / (tp + 1.0e-6)
    return [dq, sq, dq * sq], [paired_true, paired_pred, unpaired_true, unpaired_pred]


def _fast_dice_2(tab):
    tab.check_contiguous()
    if tab.inter.size == 0:
        raise ZeroDivisionError("division by zero")
    ta, pa = tab.areas()
    return np.float64(2 * int(tab.inter.sum())) / np.float64(int((ta + pa).sum()))


def _dice_1(tab):
    inter = np.int64(tab.inter.sum())
    denom = np.int64(tab.c[tab.t > 0].sum() + tab.c[tab.p > 0].sum())
    return 2.0 * inter / denom


def _dice_2(tab):
    if not tab.t_has0 or not tab.p_has0:
        raise ValueError("list.remove(x): x not in list")
    if tab.inter.size == 0:
        raise ZeroDivisionError("division by zero")
    ta = tab.tarea[np.searchsorted(tab.tid, tab.it)]
    pa = tab.parea[np.searchsorted(tab.pid, tab.ip)]
    return np.float64(2 * int(tab.inter.sum())) / np.float64(int((ta + pa).sum()))


# --------------------------------------------------------------------------------------- reference API
def get_fast_aji(true, pred):
    """AJI as distributed with MoNuSeg: every true instance is paired with the prediction of highest IoU (a
    prediction may be used several times).  Ids must be contiguous (`remap_label`)."""
    return _aji(_table(true, pred))


def get_fast_aji_plus(true, pred):
    """AJI+: a unique (Munkres) pairing of true and predicted instances; the unpaired ones add to the union.
    Ids must be contiguous (`remap_label`).  Needs N_true x N_pred float64 of host memory."""
    return _aji_plus(_table(true, pred))


def get_fast_pq(true, pred, match_iou=0.5):
    """Panoptic quality.  Returns [dq, sq, pq], [paired_true, paired_pred, unpaired_true, unpaired_pred].
    Pairs need IoU > match_iou; below 0.5 they come from a Munkres assignment (N_true x N_pred float64 of host
    memory).  Ids must be contiguous (`remap_label`)."""
    assert match_iou >= 0.0, "Cant' be negative"
    true, pred = np.asarray(true), np.asarray(pred)
    return _pq(_table(true, pred), match_iou, (true.dtype, pred.dtype))


def get_fast_dice_2(true, pred):
    """Ensemble dice over overlapping instance pairs.  Ids must be contiguous (`remap_label`)."""
    return _fast_dice_2(_table(true, pred))


def get_dice_1(true, pred):
    """Dice of the binary foreground masks."""
    return _dice_1(_table(true, pred))


def get_dice_2(true, pred):
    """Ensemble dice (Computational Precision Medicine challenge); any non-negative ids, background 0 required."""
    return _dice_2(_table(true, pred))


def remap_label(pred, by_size=False):
    """Renames the instance ids to 1..N in ascending id order, or by descending area (ties in ascending id
    order) with by_size.  Returns `pred` itself when it has no instance, else an int32 map."""
    arr = np.asarray(pred)
    tab = _table(arr, None)
    if not tab.t_has0:
        raise ValueError("list.remove(x): x not in list")
    if tab.tid.size == 0:
        return pred
    order = np.arange(tab.tid.size)
    if by_size:
        order = np.lexsort((tab.tid, -tab.tarea))  # stable descending sort by area
    new_id = np.empty(tab.tid.size, np.int32)
    new_id[order] = np.arange(1, tab.tid.size + 1, dtype=np.int32)
    out = np.zeros(arr.shape, np.int32)
    fg = arr != 0
    out[fg] = new_id[np.searchsorted(tab.tid, arr[fg])]
    return out


def pair_coordinates(setA, setB, radius):
    """Unique pairing of the points of setB with those of setA (Munkres on the Euclidean distance matrix) that
    keeps pairs at most `radius` apart.  Returns (pairing [K,2] indices into A and B, unpairedA, unpairedB)."""
    dist = cdist(setA, setB, metric="euclidean")
    ia, ib = linear_sum_assignment(dist)
    near = dist[ia, ib] <= radius
    ia, ib = ia[near], ib[near]
    pairing = np.stack([ia, ib], axis=-1)
    return pairing, np.delete(np.arange(setA.shape[0]), ia), np.delete(np.arange(setB.shape[0]), ib)
