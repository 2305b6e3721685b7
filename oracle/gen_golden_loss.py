"""Generates tests/golden/loss_cases.npz by running the UNMODIFIED reference loss functions (xentropy_loss, dice_loss,
mse_loss, msge_loss of models/hovernet/utils.py, applied as run_desc.py train_step applies them, with opt.py's
weights) from /root/reference on the CPU, in float32.

Run in the build container only (the GPU box has no /root/reference):  python -m oracle.gen_golden_loss

Stubs, none of which changes what is measured:
* `matplotlib` (imported by utils.py for its colour maps, unused by the loss functions) is an empty module;
* utils.py's `torch` is a proxy of torch whose `arange` drops the `device="cuda"` that get_sobel_kernel hard-codes,
  so the Sobel kernels are built on the CPU; every other attribute is torch's own.

Every input is rebuilt from seeds, so the file regenerates equal.  Per case k:
  probs_<k> float32 [B,h,w,4+nt]  [np p0, np p1, hv x, hv y, tp p0..] (the layout of hvn_valid_loss's probs)
  fg_<k>    uint8 [B,h,w]          the NP target (inst > 0)
  hv_<k>    float32 [B,h,w,2]      the HV target
  tp_<k>    int32 [B,h,w]          the type target (nt > 0 only)
and in `results` (JSON) nt and every loss_<branch>_<term> and overall_loss value the reference returned.
"""
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden")

# name, B, h, w, nr_types, kind
CASES = [
    ("c80_t5", 1, 80, 80, 5, "blobs"),
    ("c164_t0", 1, 164, 164, 0, "blobs"),
    ("c7x5_b33_t6", 33, 7, 5, 6, "blobs"),
    ("c3x3_t5", 4, 3, 3, 5, "blobs"),
    ("c1x1_t0", 2, 1, 1, 0, "all_fg"),
    ("no_fg_t0", 2, 20, 24, 0, "no_fg"),
    ("no_fg_t6", 1, 17, 13, 6, "no_fg"),
    ("all_fg_t5", 2, 16, 16, 5, "all_fg"),
    ("clamp_t6", 2, 12, 12, 6, "clamp"),
    ("absent_t6", 2, 24, 20, 6, "absent"),
]


def _import_ref():
    mpl = types.ModuleType("matplotlib")
    mpl.cm = types.ModuleType("matplotlib.cm")
    for name, mod in (("matplotlib", mpl), ("matplotlib.cm", mpl.cm)):
        sys.modules.setdefault(name, mod)
    sys.path.insert(0, REF)
    import torch
    from models.hovernet import utils

    class _CpuTorch:
        def __getattr__(self, name):
            return getattr(torch, name)

        @staticmethod
        def arange(*a, **k):
            k.pop("device", None)
            return torch.arange(*a, **k)

    utils.torch = _CpuTorch()
    return torch, utils


def _softmax(z):
    e = np.exp(z - z.max(-1, keepdims=True))
    return (e / e.sum(-1, keepdims=True)).astype(np.float32)


def make_case(B, h, w, nt, kind, seed):
    from scipy import ndimage
    rng = np.random.default_rng(seed)
    noise = ndimage.gaussian_filter(rng.normal(size=(B, h + 8, w + 8)), (0, 2, 2))[:, 4:-4, 4:-4]
    fg = (noise > 0).astype(np.uint8)
    if kind == "no_fg":
        fg[:] = 0
    elif kind == "all_fg":
        fg[:] = 1
    p_np = _softmax(rng.normal(0, 2, (B, h, w, 2)) + 2.0 * np.stack([1 - fg, fg], -1))
    hv = (np.round(rng.uniform(-1, 1, (B, h, w, 2)) * 64) / 64 * fg[..., None]).astype(np.float32)
    p_hv = (hv + rng.normal(0, 0.3, (B, h, w, 2))).astype(np.float32)
    tp = np.where(fg > 0, rng.integers(1, max(nt, 2), (B, h, w)), 0).astype(np.int32) if nt else None
    p_tp = _softmax(rng.normal(0, 2, (B, h, w, nt))) if nt else np.zeros((B, h, w, 0), np.float32)
    if kind == "clamp":  # one-hot predictions: exactly 0 and 1, a quarter of them wrong
        wrong = rng.random((B, h, w)) < 0.25
        pn = np.where(wrong, 1 - fg, fg)
        p_np = np.stack([1 - pn, pn], -1).astype(np.float32)
        pt = np.where(rng.random((B, h, w)) < 0.25, rng.integers(0, nt, (B, h, w)), tp)
        p_tp = np.eye(nt, dtype=np.float32)[pt]
    if kind == "absent":  # class 3 exactly 0 in the prediction and never in the target
        p_tp[..., 3] = 0
        p_tp = (p_tp / p_tp.sum(-1, keepdims=True)).astype(np.float32)
        tp[tp == 3] = 4
    probs = np.concatenate([p_np, p_hv, p_tp], -1).astype(np.float32)
    return probs, fg, hv, tp


def reference_loss(torch, utils, probs, fg, hv, tp):
    """train_step's loop over branches and opt.py's weights, on CPU float32 tensors."""
    F = torch.nn.functional
    nt = probs.shape[-1] - 4
    P = torch.from_numpy(probs)
    true_np = torch.from_numpy(fg.astype(np.int64))
    true_np_onehot = F.one_hot(true_np, num_classes=2).type(torch.float32)
    true_dict = {"np": true_np_onehot, "hv": torch.from_numpy(hv)}
    pred_dict = {}
    if nt:
        true_dict["tp"] = F.one_hot(torch.from_numpy(tp.astype(np.int64)), num_classes=nt).type(torch.float32)
        pred_dict["tp"] = P[..., 4:]
    pred_dict["np"] = P[..., 0:2]
    pred_dict["hv"] = P[..., 2:4]
    funcs = {"bce": utils.xentropy_loss, "dice": utils.dice_loss, "mse": utils.mse_loss, "msge": utils.msge_loss}
    opts = {"np": {"bce": 1, "dice": 1}, "hv": {"mse": 1, "msge": 1}, "tp": {"bce": 1, "dice": 1}}
    out, loss = {}, 0
    for branch in pred_dict:
        for name, weight in opts[branch].items():
            args = [true_dict[branch], pred_dict[branch]]
            if name == "msge":
                args.append(true_np_onehot[..., 1])
            term = funcs[name](*args)
            out["loss_%s_%s" % (branch, name)] = term.item()
            loss += weight * term
    out["overall_loss"] = loss.item()
    return out


def main():
    torch, utils = _import_ref()
    arrays, results = {}, {}
    for i, (name, B, h, w, nt, kind) in enumerate(CASES):
        probs, fg, hv, tp = make_case(B, h, w, nt, kind, seed=100 + i)
        arrays["probs_" + name], arrays["fg_" + name], arrays["hv_" + name] = probs, fg, hv
        if nt:
            arrays["tp_" + name] = tp
        results[name] = dict(nt=nt, **reference_loss(torch, utils, probs, fg, hv, tp))
    arrays["results"] = np.array(json.dumps(results, indent=1))
    np.savez_compressed(os.path.join(OUT, "loss_cases.npz"), **arrays)
    print(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
