"""Drop-in for reference `compute_stats.py`: dataset-level nuclei metrics from directories of `.mat` files (the
format `infer/tile.py` writes: `inst_map`, `inst_centroid`, `inst_type`).

    python -m hover_net_b200.compute_stats --mode instance --pred_dir PRED/ --true_dir TRUE/
    python -m hover_net_b200.compute_stats --mode type --pred_dir PRED/ --true_dir TRUE/

Instance mode makes one device pair-table call per image (`metrics.stats_utils.pair_table`) on the raw maps.
`remap_label(by_size=False)` is an order-preserving renaming of the ids, so the table of the raw maps with renamed
ids gives all six metrics; the remapped maps are never built.  Values and printed lines match the reference.
"""
import argparse
import glob
import os

import numpy as np
import scipy.io as sio

from .metrics import stats_utils as S


def run_nuclei_type_stat(pred_dir, true_dir, type_uid_list=None, exhaustive=True):
    """Detection F1, type accuracy and per-type F1 from `inst_centroid` / `inst_type` (centroids paired within 12
    px).  Note that the files are matched as `pred_dir + "*.mat"`, so pred_dir needs its trailing separator.
    Prints the results; returns None."""
    names = sorted(glob.glob(pred_dir + "*.mat"))

    def load(path):
        info = sio.loadmat(path)
        cen = info["inst_centroid"].astype("float32")
        typ = info["inst_type"].astype("int32")
        if cen.shape[0] == 0:  # an image without instances contributes one placeholder point of type 0 at (0, 0)
            return np.array([[0, 0]]), np.array([0])
        return cen, typ[:, 0]

    paired, unp_true, unp_pred, true_types, pred_types = [], [], [], [], []
    n_true = n_pred = 0  # instances of the images before this one
    for path in names:
        base = os.path.basename(path).split(".")[0]
        t_cen, t_typ = load(os.path.join(true_dir, base + ".mat"))
        p_cen, p_typ = load(os.path.join(pred_dir, base + ".mat"))
        pairing, ut, up = S.pair_coordinates(t_cen, p_cen, 12)
        if pairing.shape[0] != 0:
            paired.append(pairing + np.array([n_true, n_pred]))
        unp_true.append(ut + n_true)
        unp_pred.append(up + n_pred)
        true_types.append(t_typ)
        pred_types.append(p_typ)
        n_true += t_typ.shape[0]
        n_pred += p_typ.shape[0]

    paired = np.concatenate(paired, axis=0)
    true_types = np.concatenate(true_types, axis=0)
    pred_types = np.concatenate(pred_types, axis=0)
    pt = true_types[paired[:, 0]]
    pp = pred_types[paired[:, 1]]
    ut = true_types[np.concatenate(unp_true, axis=0)]
    up = pred_types[np.concatenate(unp_pred, axis=0)]

    def f1_type(type_id, w):
        sel = (pt == type_id) | (pp == type_id)
        st, sp = pt[sel], pp[sel]
        tp_dt = ((st == type_id) & (sp == type_id)).sum()
        tn_dt = ((st != type_id) & (sp != type_id)).sum()
        fp_dt = ((st != type_id) & (sp == type_id)).sum()
        fn_dt = ((st == type_id) & (sp != type_id)).sum()
        if not exhaustive:
            fp_dt -= (st == -1).sum()
        fp_d = (up == type_id).sum()
        fn_d = (ut == type_id).sum()
        return (2 * (tp_dt + tn_dt)) / (2 * (tp_dt + tn_dt) + w[0] * fp_dt + w[1] * fn_dt + w[2] * fp_d + w[3] * fn_d)

    tp_d, fp_d, fn_d = pp.shape[0], up.shape[0], ut.shape[0]
    tp_tn_dt = (pp == pt).sum()
    fp_fn_dt = (pp != pt).sum()
    if not exhaustive:
        fp_fn_dt -= (pt == -1).sum()
    acc_type = tp_tn_dt / (tp_tn_dt + fp_fn_dt)
    f1_d = 2 * tp_d / (2 * tp_d + 1 * fp_d + 1 * fn_d)

    if type_uid_list is None:
        type_uid_list = np.unique(true_types).tolist()
    results = [f1_d, acc_type] + [f1_type(u, [2, 2, 1, 1]) for u in type_uid_list]
    print(_fmt(np.array(results)))
    return


def _fmt(a):
    return np.array2string(a, formatter={"float": "{: 0.5f}".format})


def inst_metrics(tab_raw):
    """[dice_1, aji, dq, sq, pq, aji_plus] of one image from the pair table of its raw (pred, true) ids, in the
    order and with the exceptions of the reference's per-image loop."""
    if not tab_raw.p_has0 or not tab_raw.t_has0:  # remap_label(pred), then remap_label(true)
        raise ValueError("list.remove(x): x not in list")
    tab = tab_raw.renamed()
    pq = S._pq(tab, 0.5, (np.int32, np.int32))[0]
    return [S._dice_1(tab), S._aji(tab), pq[0], pq[1], pq[2], S._aji_plus(tab)]


def run_nuclei_inst_stat(pred_dir, true_dir, print_img_stats=False, ext=".mat"):
    """Per-image DICE, AJI, DQ, SQ, PQ and AJI+ of the `inst_map`s in pred_dir against those in true_dir (same
    basenames).  Prints pred_dir and the averages; returns the [6, n_images] array."""
    print(pred_dir)
    names = sorted(glob.glob("%s/*%s" % (pred_dir, ext)))
    metrics = [[], [], [], [], [], []]
    for path in names:
        base = os.path.basename(path).split(".")[0]
        true = sio.loadmat(os.path.join(true_dir, base + ".mat"))["inst_map"].astype("int32")
        pred = sio.loadmat(os.path.join(pred_dir, base + ".mat"))["inst_map"].astype("int32")
        rows, _ = S.pair_table(true, pred)
        for k, v in enumerate(inst_metrics(S._Pairs(rows, true.size))):
            metrics[k].append(v)
        if print_img_stats:
            print(base, end="\t")
            for scores in metrics:
                print("%f " % scores[-1], end="  ")
            print()
    metrics = np.array(metrics)
    print(_fmt(np.mean(metrics, axis=-1)))
    return metrics


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", nargs="?", default="instance", const="instance",
                    help="`instance` for nuclei instance segmentation, `type` for nuclei type classification")
    ap.add_argument("--pred_dir", nargs="?", default="", const="", help="directory of predicted .mat files")
    ap.add_argument("--true_dir", nargs="?", default="", const="", help="directory of ground-truth .mat files")
    args = ap.parse_args(argv)
    if args.mode == "instance":
        run_nuclei_inst_stat(args.pred_dir, args.true_dir, print_img_stats=False)
    if args.mode == "type":
        run_nuclei_type_stat(args.pred_dir, args.true_dir)


if __name__ == "__main__":
    main()
