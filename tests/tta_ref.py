"""Host restatement of test-time augmentation (DESIGN.md §4.5): the eight dihedral views, the map that brings a view's
output back to the input's frame, and the fp32 merge in the engine's summation order.

Arrays are [..., H, W, C] (a batch axis in front is optional); the HV vector is in the last two channels, h (x-offset,
positive to the right) then v (y-offset, positive down)."""
import numpy as np

NVIEWS = 8


def view(x, t):
    """V_t(x) = rot90(flip(x, 1) if f else x, k) over the two spatial axes, k = t % 4, f = t // 4."""
    k, f = t % 4, t // 4
    return np.ascontiguousarray(np.rot90(np.flip(x, -2) if f else x, k, axes=(-3, -2)))


def unview(y, t, vector=True):
    """Brings the output y_t of view t back: rot90(y_t, -k), then flip(., 1) if f; with vector=True the last two
    channels are then mapped (h, v) <- (-v, h) k times and h <- -h if f."""
    k, f = t % 4, t // 4
    u = np.rot90(y, -k, axes=(-3, -2))
    if f:
        u = np.flip(u, -2)
    u = np.array(u, copy=True)
    if vector:
        h, v = u[..., -2].copy(), u[..., -1].copy()
        for _ in range(k):
            h, v = -v, h
        if f:
            h = -h
        u[..., -2], u[..., -1] = h, v
    return u


def views(batch):
    """[n,H,W,3] -> [8n,H,W,3], view t of input i in slot 8i + t (the engine's order)."""
    return np.stack([view(batch[i], t) for i in range(batch.shape[0]) for t in range(NVIEWS)])


def oracle_tta(x, sd, mode, nt, device="cuda"):
    """TTA over the fp64 oracle network (oracle/hovernet_torch.forward_logits) on uint8 patches x [n,H,W,3], sd the
    numpy checkpoint: per view the NP / TP softmax probabilities and the raw HV, brought back and averaged; TP is the
    argmax of the mean probability.  Returns float64 [n,h,w,C] in the engine's channel order."""
    import torch
    from oracle import hovernet_torch as O
    tsd = {k: v.to(device=device, dtype=torch.float64) for k, v in O.to_torch_state_dict(sd).items() if v.dim() > 0}
    per_view = []
    for t in range(NVIEWS):
        xt = torch.as_tensor(view(x, t)).to(device).double().permute(0, 3, 1, 2).contiguous()
        with torch.no_grad():
            p = {k: v.permute(0, 2, 3, 1) for k, v in O.forward_logits(xt, tsd, mode, nt).items()}
            cols = [torch.softmax(p["tp"], -1)] if nt else []
            cols += [torch.softmax(p["np"], -1)[..., 1:], p["hv"]]
            per_view.append(unview(torch.cat(cols, -1).cpu().numpy(), t))
    mean = sum(per_view) / float(NVIEWS)
    out = mean[..., -3:]
    if nt:
        out = np.concatenate([np.argmax(mean[..., :nt], -1)[..., None].astype(np.float64), out], -1)
    return out


def merge(per_view):
    """per_view: [8, ..., C] outputs of the eight views of the same inputs (view t at index t).  Brings each back and
    averages in fp32 in view order: s = u_0; s += u_1; ...; s += u_7; s *= 0.125."""
    s = unview(np.asarray(per_view[0], np.float32), 0)
    for t in range(1, NVIEWS):
        s += unview(np.asarray(per_view[t], np.float32), t)
    s *= np.float32(0.125)
    return s
