"""Command line of the reference `run_infer.py` (SURVEY.md row f1) over the libhvn engine.

    python -m hover_net_b200.run_infer [options] tile --input_dir=<path> --output_dir=<path> [...]
    python -m hover_net_b200.run_infer [options] wsi  --input_dir=<path> --output_dir=<path> [...]

Same option names, defaults and `method_args` / `run_args` dictionaries as reference
`run_infer.py:1-186` (docopt there, argparse here -- docopt is not a dependency of this repo);
`--option=value` and `--option value` are both accepted.  Differences that follow from the engine:
one process drives one GPU (`--gpu` takes the first id of the list unless the process was launched by
torchrun, where LOCAL_RANK picks the device and files / patches are sharded over the ranks), and
`--nr_inference_workers` / `--nr_post_proc_workers` are accepted and ignored (no CPU stage is left).

Extension the reference CLI lacks: `--precision {highest,high}` (default `highest`) picks the convolution operand
precision.  `highest` forms fp32-grade products (fp16 hi + lo operands); `high` stores every activation and weight
that feeds a convolution as one fp16 value and forms one product per multiply-accumulate, with fp32 accumulation --
the operand precision the reference itself gets from PyTorch's default TF32 convolutions on this GPU -- for a third of
the tensor-core work.  A non-default value is passed to `create_model` through `method_args["method"]["model_args"]`.

Extension the reference CLI lacks: `--tta` (test-time augmentation) runs every patch as its eight dihedral views
(4 rotations x optional mirror) and averages their maps on the device, the HV vectors mapped back to the patch's
frame, before post-processing: eight times the network work.  When given, `"tta": True` is added to `model_args`;
tile and WSI modes take it from the model.

Extension the reference CLI lacks: `--save_features` (tile and wsi) measures every nucleus on the device -- area,
contour and convex areas, perimeter, solidity, circularity, ellipse axes, eccentricity, orientation, maximum Feret
diameter, mean and standard deviation of each RGB channel, and the mean NP probability -- and adds them to each JSON
record as "features" (tile mode also to the `.mat` as `inst_features` / `inst_feature_names`).  Without it every output
is what the reference writes.
"""
import argparse
import logging
import os

VERSION = "HoVer-Net H100 Inference v1.0"


def _top_parser():
    ap = argparse.ArgumentParser(prog="run_infer.py", add_help=False, allow_abbrev=False)
    ap.add_argument("-h", "--help", action="store_true")
    ap.add_argument("--version", action="store_true")
    ap.add_argument("--gpu", default="0")
    ap.add_argument("--nr_types", default="0")
    ap.add_argument("--type_info_path", default="")
    ap.add_argument("--model_path", default=None)
    ap.add_argument("--model_mode", default="fast")
    ap.add_argument("--nr_inference_workers", default="8")
    ap.add_argument("--nr_post_proc_workers", default="16")
    ap.add_argument("--batch_size", default="32")
    ap.add_argument("--precision", default="highest", choices=["highest", "high"])
    ap.add_argument("--tta", action="store_true")
    return ap


def _tile_parser():
    ap = argparse.ArgumentParser(prog="run_infer.py tile", allow_abbrev=False)
    ap.add_argument("--input_dir", required=True)
    ap.add_argument("--output_dir", required=True)
    ap.add_argument("--mem_usage", default="0.2")
    ap.add_argument("--draw_dot", action="store_true")
    ap.add_argument("--save_qupath", action="store_true")
    ap.add_argument("--save_raw_map", action="store_true")
    ap.add_argument("--save_features", action="store_true")
    return ap


def _wsi_parser():
    ap = argparse.ArgumentParser(prog="run_infer.py wsi", allow_abbrev=False)
    ap.add_argument("--input_dir", required=True)
    ap.add_argument("--output_dir", required=True)
    ap.add_argument("--cache_path", default="cache")
    ap.add_argument("--input_mask_dir", default=None)
    ap.add_argument("--proc_mag", default="40")
    ap.add_argument("--ambiguous_size", default="128")
    ap.add_argument("--chunk_shape", default="10000")
    ap.add_argument("--tile_shape", default="2048")
    ap.add_argument("--save_thumb", action="store_true")
    ap.add_argument("--save_mask", action="store_true")
    ap.add_argument("--save_features", action="store_true")
    return ap


def parse(argv, nr_gpus=1):
    """argv (without the program name) -> (sub_cmd, method_args, run_args, gpu_list).
    sub_cmd is None when only help / version was asked for."""
    # options first, then the command and its own options (docopt `options_first=True`)
    split = next((i for i, a in enumerate(argv) if a in ("tile", "wsi")), None)
    top_argv = argv if split is None else argv[:split]
    args = _top_parser().parse_args(top_argv)
    if split is None or args.help or args.version:
        return None, None, None, args.gpu
    sub_cmd = argv[split]
    sub = (_tile_parser() if sub_cmd == "tile" else _wsi_parser()).parse_args(argv[split + 1:])
    if args.model_path is None:
        raise Exception("A model path must be supplied as an argument with --model_path.")
    nr_types = int(args.nr_types) if int(args.nr_types) > 0 else None
    method_args = {
        "method": {
            "model_args": {"nr_types": nr_types, "mode": args.model_mode},
            "model_path": args.model_path,
        },
        "type_info_path": None if args.type_info_path == "" else args.type_info_path,
    }
    if args.precision != "highest":  # the default leaves model_args exactly as the reference builds them
        method_args["method"]["model_args"]["precision"] = args.precision
    if args.tta:
        method_args["method"]["model_args"]["tta"] = True
    run_args = {
        "batch_size": int(args.batch_size) * max(1, nr_gpus),
        "nr_inference_workers": int(args.nr_inference_workers),
        "nr_post_proc_workers": int(args.nr_post_proc_workers),
    }
    if args.model_mode == "fast":
        run_args["patch_input_shape"], run_args["patch_output_shape"] = 256, 164
    else:
        run_args["patch_input_shape"], run_args["patch_output_shape"] = 270, 80
    if sub_cmd == "tile":
        run_args.update({
            "input_dir": sub.input_dir, "output_dir": sub.output_dir, "mem_usage": float(sub.mem_usage),
            "draw_dot": sub.draw_dot, "save_qupath": sub.save_qupath, "save_raw_map": sub.save_raw_map,
        })
    else:
        run_args.update({
            "input_dir": sub.input_dir, "output_dir": sub.output_dir, "input_mask_dir": sub.input_mask_dir,
            "cache_path": sub.cache_path, "proc_mag": int(sub.proc_mag), "ambiguous_size": int(sub.ambiguous_size),
            "chunk_shape": int(sub.chunk_shape), "tile_shape": int(sub.tile_shape),
            "save_thumb": sub.save_thumb, "save_mask": sub.save_mask,
        })
    if sub.save_features:  # the default leaves run_args exactly as the reference builds them
        run_args["save_features"] = True
    return sub_cmd, method_args, run_args, args.gpu


def main(argv=None):
    import sys
    argv = list(sys.argv[1:] if argv is None else argv)
    sub_cmd, method_args, run_args, gpu_list = parse(argv)
    if sub_cmd is None:
        if "--version" in argv:
            print(VERSION)
        else:
            print(__doc__)
            _top_parser().print_help()
            _tile_parser().print_help()
            _wsi_parser().print_help()
        return 0
    logging.basicConfig(level=logging.INFO, format="|%(asctime)s.%(msecs)03d| [%(levelname)s] %(message)s",
                        datefmt="%Y-%m-%d|%H:%M:%S")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:  # launched by torchrun: one rank per GPU, work sharded by the drivers
        import torch
        import torch.distributed as dist
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        method_args["method"]["model_args"]["device"] = local
    else:
        method_args["method"]["model_args"]["device"] = int(str(gpu_list).split(",")[0])
    if sub_cmd == "tile":
        from .infer.tile import InferManager
        InferManager(**method_args).process_file_list(run_args)
    else:
        from .infer.wsi import InferManager
        InferManager(**method_args).process_wsi_list(run_args)
    if world > 1:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
