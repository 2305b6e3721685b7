"""Benchmark of tile mode over many images on one GPU: the grouped `process_file_list` against today's one-file-at-a-time
loop, writers included, and the device path alone.

Workloads (seeded synthetic images written as PNG to a temporary directory, seeded checkpoints):
* pannuke: 256 images of 256 x 256, `fast` mode, nr_types 6 (2 x 2 patches each);
* consep: 16 images of 1000 x 1000, `original` mode, nr_types 5 (13 x 13 patches each).

Arms, alternated in one process over --repeats rounds (images/s, median and spread over the rounds):
* serial: the loop `process_file_list` ran before groups -- read a file, `infer_image`, write its files -- restated here;
* grouped: `process_file_list` with mem_usage 0.2 (every file fits one group: cross-image batching, no overlap);
* grouped_8: `process_file_list` with mem_usage set so that the RAM rule cuts about 8 groups: the device runs a group
  while the previous group's files are written and the next group's files are read;
* device-only: an `infer_image` loop against one `infer_images` call on the images already in memory.
The card name and power limit are read in the same run.

usage: python tools/bench_tiles.py --out DIR [--repeats N] [--batch B]
"""
import argparse
import glob
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hover_net_b200 import synth  # noqa: E402

WORKLOADS = {"pannuke": dict(n=256, size=256, mode="fast", nt=6, win=256, msk=164),
             "consep": dict(n=16, size=1000, mode="original", nt=5, win=270, msk=80)}


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def _image(size, seed):
    k = -(-size // 256)
    t = synth.make_patches(k * k, 256, seed=seed)
    big = np.concatenate([np.concatenate(list(t[r * k:(r + 1) * k]), 1) for r in range(k)], 0)
    return np.ascontiguousarray(big[:size, :size])


def _serial(mgr, run_args):
    """process_file_list as it ran one file at a time: read, infer_image, write."""
    import cv2
    from hover_net_b200.infer import tile
    for variable, value in run_args.items():
        setattr(mgr, variable, value)
    for sub in ("json", "mat", "overlay"):
        tile._rm_n_mkdir(mgr.output_dir + "/%s/" % sub)
    for path in sorted(glob.glob(mgr.input_dir + "/*")):
        img = cv2.cvtColor(cv2.imread(path), cv2.COLOR_BGR2RGB)
        pred_map, pred_inst, info = mgr.infer_image(img)
        mgr._write_files([(path, img)], [(pred_map, pred_inst, info)])


def bench(name, w, repeats, batch):
    import cv2
    from hover_net_b200.infer.tile import InferManager
    d = tempfile.mkdtemp(prefix="bench_tiles_")
    imgs = [_image(w["size"], 500 + i) for i in range(w["n"])]
    os.makedirs(d + "/in")
    for i, img in enumerate(imgs):
        cv2.imwrite("%s/in/%04d.png" % (d, i), cv2.cvtColor(img, cv2.COLOR_RGB2BGR))
    mgr = InferManager(method={"model_args": {"nr_types": w["nt"], "mode": w["mode"]},
                               "model_path": synth.make_state_dict(w["mode"], w["nt"], seed=0)}, type_info_path=None)
    run_args = {"batch_size": batch, "nr_inference_workers": 0, "nr_post_proc_workers": 0,
                "patch_input_shape": w["win"], "patch_output_shape": w["msk"], "input_dir": d + "/in",
                "mem_usage": 0.2, "draw_dot": False, "save_qupath": False, "save_raw_map": False}
    mgr.patch_input_shape, mgr.patch_output_shape, mgr.batch_size = w["win"], w["msk"], batch
    import psutil
    from hover_net_b200.infer import tile
    ram = tile._file_cost((w["size"], w["size"], 3), w["win"], w["msk"])[0]
    mem8 = min(0.99, (ram * (w["n"] // 8) + ram // 2) / psutil.virtual_memory().available)
    groups = []
    real = tile._groups

    def counted(items, costs, budgets):
        for g in real(items, costs, budgets):
            groups.append(len(g))
            yield g
    tile._groups = counted
    arms = {"serial": lambda: _serial(mgr, dict(run_args, output_dir=d + "/out_serial")),
            "grouped": lambda: mgr.process_file_list(dict(run_args, output_dir=d + "/out_grouped")),
            "grouped_8": lambda: mgr.process_file_list(dict(run_args, mem_usage=mem8, output_dir=d + "/out_grouped_8")),
            "device_serial": lambda: [mgr.infer_image(img) for img in imgs],
            "device_grouped": lambda: mgr.infer_images(imgs)}
    for k, f in arms.items():  # warm-up: plans, arenas; the group sizes each file arm formed
        groups.clear()
        f()
        if k.startswith("grouped"):
            w = dict(w, **{"groups_" + k: list(groups)})
    t = {k: [] for k in arms}
    groups.clear()
    for _ in range(repeats):
        for k, f in arms.items():
            t0 = time.perf_counter()
            f()
            t[k].append(time.perf_counter() - t0)
    # the file arms wrote the same files (the .mat header carries its creation time)
    same = True
    for sub in ("mat", "json", "overlay"):
        for p in sorted(glob.glob(d + "/out_serial/%s/*" % sub)):
            a = open(p, "rb").read()
            for arm in ("out_grouped", "out_grouped_8"):
                b = open(p.replace("out_serial", arm), "rb").read()
                same = same and a[116 if sub == "mat" else 0:] == b[116 if sub == "mat" else 0:]
    n = w["n"]
    res = {"workload": name, **{k: v for k, v in w.items()}, "batch": batch, "repeats": repeats,
           "files_identical": bool(same)}
    for k, v in t.items():
        ips = sorted(n / x for x in v)
        res[k] = {"images_per_s_median": float(np.median(ips)), "images_per_s_min": ips[0], "images_per_s_max": ips[-1]}
    tile._groups = real
    mgr.net.ctx.close()
    import shutil
    shutil.rmtree(d, ignore_errors=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    out = {"card": _card(), "results": []}
    for name, w in WORKLOADS.items():
        r = bench(name, w, a.repeats, a.batch)
        print(json.dumps(r), flush=True)
        out["results"].append(r)
    out["card_after"] = _card()
    with open(os.path.join(a.out, "h100_bench_tiles.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({"card": out["card"]}))


if __name__ == "__main__":
    main()
