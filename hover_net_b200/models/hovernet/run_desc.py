"""Drop-in for reference `models/hovernet/run_desc.py`: `infer_step` (:171-197), `valid_step` (:113-167) and
`proc_valid_step_output` (:263-344, scalars only), plus `loss_scalars`: the loss values `train_step` (:12-109)
tracks, from the sums of hvn_valid_loss."""
import numpy as np


def _as_u8(batch_data):
    x = batch_data
    if hasattr(x, "detach"):  # torch tensor from the default collate (infer_loader.py:65-72)
        x = x.detach().cpu().numpy()
    x = np.asarray(x)
    if x.dtype != np.uint8:
        # the reference casts to float32 and divides by 255; image patches are integral 0..255
        if not np.array_equal(x, np.round(x)) or x.min() < 0 or x.max() > 255:
            raise ValueError("infer_step expects integral RGB values in 0..255")
        x = x.astype(np.uint8)
    return np.ascontiguousarray(x)


def infer_step(batch_data, model):
    """uint8 NHWC [B,H,W,3] -> np.float32 [B,h,w,C] ([tp?, np, hv_x, hv_y])."""
    net = getattr(model, "module", model)
    return net.ctx.forward(_as_u8(batch_data))


def infer_step_fused(batch_data, model, return_pred=True):
    """infer_step + post_proc.process on every patch without the maps leaving the device.
    Returns (pred or None, inst [B,h,w] int32, table [B,max_rows,10] int64, n_rows [B])."""
    net = getattr(model, "module", model)
    return net.ctx.forward_postproc(_as_u8(batch_data), want_pred=return_pred)


def _host(x):
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def valid_step(batch_data, run_info):
    """Reference `valid_step`: batch_data {"img" [B,H,W,3], "np_map" [B,h,w], "hv_map" [B,h,w,2], "tp_map"
    [B,h,w] with types}, run_info = (run_info, state_info) with run_info["net"]["desc"] the model.  Returns the
    reference's {"raw": {"imgs", "true_np", "true_hv", "prob_np", "pred_hv", ["true_tp", "pred_tp"]}}.  Unlike the
    reference, a batch of one patch keeps its batch axis (the reference's squeeze drops it)."""
    run_info, _state_info = run_info
    net = getattr(run_info["net"]["desc"], "module", run_info["net"]["desc"])
    imgs = _as_u8(batch_data["img"])
    pred = net.ctx.forward(imgs)
    raw = {
        "imgs": _host(batch_data["img"]),
        "true_np": _host(batch_data["np_map"]).astype(np.int64),
        "true_hv": _host(batch_data["hv_map"]).astype(np.float32),
        "prob_np": np.ascontiguousarray(pred[..., -3]),
        "pred_hv": np.ascontiguousarray(pred[..., -2:]),
    }
    if net.nr_types is not None:
        raw["true_tp"] = _host(batch_data["tp_map"]).astype(np.int64)
        raw["pred_tp"] = np.ascontiguousarray(pred[..., 0])
    return {"raw": raw}


def valid_scalars(correct, inter, total, type_counts, hv_sse, nr_pixels):
    """The reference's scalars from integer counts: np_acc, np_dice, tp_dice_<k> (type_counts: [(inter_k,
    total_k)] or None), hv_mse.  The integer ratios are evaluated exactly as the reference evaluates them."""
    out = {}
    out["np_acc"] = np.int64(correct) / nr_pixels
    out["np_dice"] = 2 * np.int64(inter) / (np.int64(total) + 1.0e-8)
    for k, (ik, tk) in enumerate(type_counts or ()):
        out["tp_dice_%d" % k] = 2 * np.int64(ik) / (np.int64(tk) + 1.0e-8)
    out["hv_mse"] = hv_sse / nr_pixels
    return out


def proc_valid_step_output(raw_data, nr_types=None):
    """Reference `proc_valid_step_output`, restated on host numpy arrays with the same operations on the same
    values, so the scalars are bit-identical.  Returns {"scalar": {...}, "image": {}}: the reference's image entry
    is a matplotlib figure, and matplotlib is not a dependency of this package."""
    prob_np, true_np = raw_data["prob_np"], raw_data["true_np"]
    n = len(true_np)
    pred_np = (np.asarray(prob_np) > 0.5).astype(np.int32)
    true_np = np.asarray(true_np)
    correct = int((pred_np == true_np).sum())
    t1 = (true_np == 1).astype(np.int32)
    p1 = (pred_np == 1).astype(np.int32)
    inter, total = int((t1 * p1).sum()), int((t1 + p1).sum())
    type_counts = None
    if nr_types is not None:
        pred_tp, true_tp = np.asarray(raw_data["pred_tp"]), np.asarray(raw_data["true_tp"])
        type_counts = []
        for k in range(nr_types):
            tk = (true_tp == k).astype(np.int32)
            pk = (pred_tp == k).astype(np.int32)
            type_counts.append((int((tk * pk).sum()), int((tk + pk).sum())))
    # float32 per-patch sums accumulated in patch order, as the reference does
    sse = 0
    for i in range(n):
        d = raw_data["pred_hv"][i] - raw_data["true_hv"][i]
        sse += (d * d).sum()
    nr_pixels = n * np.size(true_np[0])
    scalar = valid_scalars(correct, inter, total, type_counts, sse, nr_pixels)
    return {"scalar": scalar, "image": {}}


# opt.py extra_info["loss"]: every term has weight 1
LOSS_OPTS = {"np": {"bce": 1, "dice": 1}, "hv": {"mse": 1, "msge": 1}, "tp": {"bce": 1, "dice": 1}}


def loss_scalars(sums, nr_pixels, loss_opts=None):
    """The reference's training loss (train_step with utils.py xentropy_loss, dice_loss, mse_loss, msge_loss) from
    the sums of `Context.valid_loss` (layout in include/hvn.h; 10 entries untyped, 11 + 3*nr_types typed) over
    nr_pixels = B*h*w output pixels.  Sums added over several batches give the loss of the set as one batch.
    Returns {"loss_<branch>_<term>": value, ..., "overall_loss": weighted sum} in train_step's order: branches tp
    (when typed), np, hv; terms in loss_opts' order (default: opt.py's weights, all 1).  Float64 throughout."""
    s = np.asarray(sums, np.float64)
    n = float(nr_pixels)
    nt = (len(s) - 11) // 3 if len(s) > 10 else 0

    def dice(i, l, r):
        return float(np.sum(1.0 - (2.0 * i + 1e-3) / (l + r + 1e-3)))

    terms = {
        "np": {"bce": s[0] / n, "dice": dice(s[1:3], s[3:5], s[5:7])},
        "hv": {"mse": s[7] / (2.0 * n), "msge": s[8] / (2.0 * s[9] + 1.0e-8)},
    }
    if nt:
        terms["tp"] = {"bce": s[10] / n,
                       "dice": dice(s[11:11 + nt], s[11 + nt:11 + 2 * nt], s[11 + 2 * nt:11 + 3 * nt])}
    opts = LOSS_OPTS if loss_opts is None else loss_opts
    out, total = {}, 0.0
    for branch in (("tp",) if nt else ()) + ("np", "hv"):
        for name, weight in opts[branch].items():
            v = float(terms[branch][name])
            out["loss_%s_%s" % (branch, name)] = v
            total += weight * v
    out["overall_loss"] = total
    return out
