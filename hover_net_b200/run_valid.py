"""Scores a checkpoint on labelled patches with the reference's validation protocol (run_train.py in "valid"
mode: `FileLoader`, `valid_step`, `proc_valid_step_output`), on one GPU.  The reference has no such command; its
scalars come out of the training loop.

Every `*.npy` patch of the --valid_dir directories (sorted, as run_train._get_datagen orders them) is centre-cropped
to the network input; each batch runs forward, targets and the counts in one device call (hvn_valid), and the
counts are summed on the host.  Prints np_acc, np_dice, tp_dice_<k> (with --nr_types) and hv_mse, the reference's
names.  hv_mse sums in float64 where the reference sums in float32.

usage: python -m hover_net_b200.run_valid --model_path CKPT --valid_dir DIR [--valid_dir DIR ...]
       [--model_mode original|fast] [--nr_types N] [--batch_size B] [--precision highest|high] [--tta] [--loss]
       [--json OUT]

--tta scores the checkpoint with test-time augmentation (the eight dihedral views of every patch, merged on the
device), so that its effect on these scalars can be measured on the user's own labelled patches.

--loss also prints the reference's training loss on these patches (train_step's loss_<branch>_<term> names and
overall_loss, opt.py's weights), after the scalars above: each batch runs hvn_valid_loss instead of hvn_valid, the
per-batch sums are added in float64, and the loss formulas are applied once to the set's sums, so the values are those
of the whole set as one batch, whatever --batch_size is.  The network runs in eval mode (running BatchNorm
statistics), so this is the validation loss: train_step evaluates the same formulas with batch statistics.  hv_mse
then comes from the loss pass's sum, equal to hvn_valid's to float64 reordering.
"""
import argparse
import ctypes
import glob
import json
import sys

import numpy as np

# the reference's config.py: network input / output shapes per mode
SHAPES = {"original": ([270, 270], [80, 80]), "fast": ([256, 256], [164, 164])}


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="validation statistics of a HoVer-Net checkpoint on .npy patches")
    ap.add_argument("--model_path", required=True)
    ap.add_argument("--model_mode", default="original", choices=sorted(SHAPES))
    ap.add_argument("--nr_types", type=int, default=0, help="number of nuclear types (0: segmentation only)")
    ap.add_argument("--valid_dir", action="append", required=True, help="directory of .npy patches (repeatable)")
    ap.add_argument("--batch_size", type=int, default=16)
    ap.add_argument("--precision", default="highest", choices=["highest", "high"])
    ap.add_argument("--tta", action="store_true", help="test-time augmentation: eight dihedral views, merged")
    ap.add_argument("--loss", action="store_true", help="also the training loss (loss_*, overall_loss) on these patches")
    ap.add_argument("--json", default=None, help="also write the scalars to this JSON file")
    return ap.parse_args(argv)


def file_list(dirs):
    out = []
    for d in dirs:
        out.extend(glob.glob("%s/*.npy" % d))
    out.sort()
    return out


def run(args):
    from .dataloader.train_loader import FileLoader
    from .models.hovernet import net_desc, run_desc, targets

    files = file_list(args.valid_dir)
    if not files:
        raise SystemExit("no .npy patches found in %s" % args.valid_dir)
    nr_types = args.nr_types or None
    input_shape, mask_shape = SHAPES[args.model_mode]
    net = net_desc.create_model(mode=args.model_mode, nr_types=nr_types, precision=args.precision, tta=args.tta)
    # checkpoint formats as in infer/base.py: an .npz of arrays or the reference's torch file with a "desc" entry
    if str(args.model_path).endswith(".npz"):
        state = dict(np.load(args.model_path))
    else:
        import torch
        state = torch.load(args.model_path, map_location="cpu")["desc"]
    net.load_state_dict(state, strict=True)
    ctx = net.ctx
    if list(ctx.out_shape(*input_shape)[:2]) != mask_shape:
        raise ValueError("network output %s is not the mask shape %s" % (ctx.out_shape(*input_shape)[:2], mask_shape))
    loader = FileLoader(files, with_type=nr_types is not None, input_shape=input_shape, mask_shape=mask_shape,
                        mode="valid", target_gen=(targets.gen_targets, {}))
    H, W = input_shape
    B = max(1, int(args.batch_size))
    # pinned host batches, reused for every call
    nbytes = B * H * W
    p_img, p_inst, p_type = ctx.malloc_host(nbytes * 3), ctx.malloc_host(nbytes * 4), ctx.malloc_host(nbytes * 4)
    try:
        img = np.ctypeslib.as_array((ctypes.c_uint8 * (nbytes * 3)).from_address(p_img))
        inst = np.ctypeslib.as_array((ctypes.c_int32 * nbytes).from_address(p_inst))
        typ = np.ctypeslib.as_array((ctypes.c_int32 * nbytes).from_address(p_type))
        img, inst, typ = img.reshape(B, H, W, 3), inst.reshape(B, H, W), typ.reshape(B, H, W)
        counts = np.zeros((3 + 2 * (nr_types or 0),), np.int64)
        sse = 0.0
        sums = 0.0
        for lo in range(0, len(files), B):
            n = min(B, len(files) - lo)
            for i in range(n):
                a, b, t = loader.load(lo + i)
                img[i], inst[i] = a, b
                if t is not None:
                    typ[i] = t
            if args.loss:
                c, s, flags, ls, _ = ctx.valid_loss(img[:n], inst[:n], typ[:n] if nr_types else None)
                sums = sums + ls
            else:
                c, s, flags = ctx.valid(img[:n], inst[:n], typ[:n] if nr_types else None)
            targets.raise_for_flags(flags, names=files[lo:lo + n])
            counts += c
            sse += s
    finally:
        for p in (p_img, p_inst, p_type):
            ctx.free_host(p)
    tc = [(counts[3 + 2 * k], counts[4 + 2 * k]) for k in range(nr_types)] if nr_types else None
    nr_pixels = len(files) * mask_shape[0] * mask_shape[1]
    scalars = run_desc.valid_scalars(counts[0], counts[1], counts[2], tc, sse, nr_pixels)
    if args.loss:
        scalars.update(run_desc.loss_scalars(sums, nr_pixels))
    return scalars


def main(argv=None):
    args = parse_args(argv)
    scalars = run(args)
    for k, v in scalars.items():
        print("%s: %s" % (k, float(v)))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({k: float(v) for k, v in scalars.items()}, f, indent=1)
    return scalars


if __name__ == "__main__":
    main(sys.argv[1:])
