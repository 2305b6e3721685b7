"""Float64 numpy restatement of the validation loss (the reference's xentropy_loss, dice_loss, mse_loss and msge_loss
of models/hovernet/utils.py, as train_step applies them), in the slot layout of hvn_valid_loss's sums.

probs [B,h,w,4+nt] = [np p0, np p1, hv x, hv y, tp p0..]; fg [B,h,w] the NP target (0/1); hv [B,h,w,2] the HV target;
tp [B,h,w] the type target (None when nt == 0)."""
import numpy as np

EPS_LO = float(np.float32(10e-8))            # torch.clamp rounds its bounds to the tensor's dtype
EPS_HI = float(np.float32(1.0 - 10e-8))


def sobel5():
    """kernel_h, kernel_v of get_sobel_kernel(5): torch.meshgrid 'ij' (h varies along rows), fp32 values."""
    r = np.arange(-2, 3, dtype=np.float32)
    h, v = np.meshgrid(r, r, indexing="ij")
    d = h * h + v * v + np.float32(1e-15)
    return (h / d).astype(np.float64), (v / d).astype(np.float64)


def xcorr5(x, k):
    """F.conv2d(x[:, None], k[None, None], padding=2)[:, 0]: cross-correlation, zero padding, x [B,h,w]."""
    B, h, w = x.shape
    p = np.zeros((B, h + 4, w + 4))
    p[:, 2:-2, 2:-2] = x
    out = np.zeros((B, h, w))
    for i in range(5):
        for j in range(5):
            out += k[i, j] * p[:, i:i + h, j:j + w]
    return out


def _ce(p, t):
    q = p / p.sum(-1, keepdims=True)
    q = np.clip(q, EPS_LO, EPS_HI)
    return float(-(t * np.log(q)).sum())


def nsums(nt):
    return 10 + (1 + 3 * nt if nt else 0)


def sums(probs, fg, hv, tp=None):
    probs = np.asarray(probs, np.float64)
    nt = probs.shape[-1] - 4
    fg = (np.asarray(fg) > 0).astype(np.float64)
    hv = np.asarray(hv, np.float64)
    out = np.zeros(nsums(nt))
    p_np = probs[..., 0:2]
    t_np = np.stack([1.0 - fg, fg], -1)
    out[0] = _ce(p_np, t_np)
    out[1:3] = (p_np * t_np).sum((0, 1, 2))
    out[3:5] = p_np.sum((0, 1, 2))
    out[5:7] = t_np.sum((0, 1, 2))
    p_hv = probs[..., 2:4]
    out[7] = ((p_hv - hv) ** 2).sum()
    kh, kv = sobel5()
    dh = xcorr5(p_hv[..., 0], kh) - xcorr5(hv[..., 0], kh)
    dv = xcorr5(p_hv[..., 1], kv) - xcorr5(hv[..., 1], kv)
    out[8] = (fg * (dh * dh + dv * dv)).sum()
    out[9] = fg.sum()
    if nt:
        tp = np.asarray(tp)
        if tp.min() < 0 or tp.max() >= nt:
            raise ValueError("type id outside 0..%d" % (nt - 1))
        p_tp = probs[..., 4:]
        t_tp = np.eye(nt)[tp]
        out[10] = _ce(p_tp, t_tp)
        out[11:11 + nt] = (p_tp * t_tp).sum((0, 1, 2))
        out[11 + nt:11 + 2 * nt] = p_tp.sum((0, 1, 2))
        out[11 + 2 * nt:11 + 3 * nt] = t_tp.sum((0, 1, 2))
    return out
