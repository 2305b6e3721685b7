"""Row f1 (tile driver): patch geometry and stitching pinned against goldens produced by the
reference's own `infer/tile.py` functions (oracle/gen_golden_tile.py); output-format checks."""
import glob
import json
import os

import numpy as np
import pytest

from hover_net_b200.infer import tile

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLD, "tile_*.npz"))))
def test_patch_geometry_and_stitching_match_reference(path):
    g = np.load(path)
    win, msk, h, w = int(g["win"]), int(g["msk"]), int(g["h"]), int(g["w"])
    img = np.random.default_rng(int(g["seed"])).integers(0, 256, (h, w, 3), dtype=np.uint8)
    padded, pinfo, corner = tile._prepare_patching(img, win, msk, True)
    assert np.array_equal(pinfo, g["patch_info"]) and list(corner) == list(g["corner"])
    assert np.array_equal(padded.shape, g["padded_shape"])
    assert np.array_equal(padded.astype(np.int64).sum((1, 2)), g["padded_rowsum"])
    data = []
    for y, x, _, _ in pinfo:
        yy, xx = np.mgrid[0:msk, 0:msk]
        data.append(np.stack([yy + y, xx + x, (yy + y) * 1000 + (xx + x), np.full_like(yy, 7)], -1).astype(np.float32))
    perm = np.random.default_rng(1).permutation(len(data))  # arrival order must not matter
    m = tile._stitch([pinfo[i] for i in perm], [data[i] for i in perm], img.shape)
    assert np.array_equal(m, g["stitched"])


def test_json_writer_format(tmp_path):
    from hover_net_b200.infer.base import InferManager
    info = {3: {"bbox": np.array([[1, 2], [5, 9]]), "centroid": np.array([4.5, 2.25]),
                "contour": np.array([[2, 1], [8, 1], [8, 4]], dtype=np.int32), "type_prob": 0.75, "type": 2},
            7: {"bbox": np.array([[0, 0], [2, 2]]), "centroid": np.array([0.5, 0.5]),
                "contour": np.array([[0, 0], [1, 0], [1, 1]], dtype=np.int32), "type_prob": None, "type": None}}
    p = str(tmp_path / "a.json")
    InferManager._save_json(None, p, info, None)
    d = json.load(open(p))
    assert d["mag"] is None and sorted(d["nuc"].keys()) == ["3", "7"]
    assert d["nuc"]["3"] == {"bbox": [[1, 2], [5, 9]], "centroid": [4.5, 2.25], "contour": [[2, 1], [8, 1], [8, 4]],
                             "type_prob": 0.75, "type": 2}
    assert d["nuc"]["7"]["type"] is None


@pytest.mark.gpu
def test_process_file_list_end_to_end(tmp_path):
    """Drive the whole tile pipeline on the device and cross-check it with the CPU oracle."""
    import cv2
    import scipy.io as sio
    import torch
    from hover_net_b200 import synth
    from hover_net_b200.infer.tile import InferManager
    from oracle import hovernet_torch as O
    from oracle import postproc_oracle as P

    mode, nt = "fast", 6
    rng = np.random.default_rng(3)
    big = np.concatenate([np.concatenate(list(synth.make_patches(2, 256, seed=40 + r)), 1) for r in range(2)], 0)
    img = big[:300, :420].copy()  # 300x420 RGB -> 2x3 patches
    os.makedirs(tmp_path / "in")
    cv2.imwrite(str(tmp_path / "in" / "tileA.png"), cv2.cvtColor(img, cv2.COLOR_RGB2BGR))
    sd = synth.make_state_dict(mode, nt, seed=0)
    mgr = InferManager(method={"model_args": {"nr_types": nt, "mode": mode}, "model_path": sd}, type_info_path=None)
    mgr.process_file_list({"batch_size": 4, "nr_inference_workers": 0, "nr_post_proc_workers": 0,
                           "patch_input_shape": 256, "patch_output_shape": 164, "input_dir": str(tmp_path / "in"),
                           "output_dir": str(tmp_path / "out"), "mem_usage": 0.1, "draw_dot": True,
                           "save_qupath": True, "save_raw_map": True})
    mat = sio.loadmat(str(tmp_path / "out" / "mat" / "tileA.mat"))
    js = json.load(open(str(tmp_path / "out" / "json" / "tileA.json")))
    assert os.path.exists(str(tmp_path / "out" / "overlay" / "tileA.png"))
    assert open(str(tmp_path / "out" / "qupath" / "tileA.tsv")).readline() == "x\ty\tclass\tname\tcolor\n"
    raw, inst = mat["raw_map"], mat["inst_map"]
    assert raw.shape == (300, 420, 4) and inst.shape == (300, 420) and inst.dtype == np.int32
    # (1) stitched float map vs the CPU oracle run over the same patch grid
    padded, pinfo, _ = tile._prepare_patching(img, 256, 164, True)
    tsd = O.to_torch_state_dict(sd)
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    outs = O.infer_step(np.stack([padded[y:y + 256, x:x + 256] for y, x, _, _ in pinfo]), tsd, mode, nt)
    ref_map = tile._stitch(list(pinfo), list(outs), img.shape)
    assert np.abs(raw[..., 1:] - ref_map[..., 1:]).max() <= 1e-4
    # (2) instances: oracle post-processing of the device-produced map must agree bit for bit
    oi, oinfo = P.process(raw, nr_types=nt, return_centroids=True)
    assert np.array_equal(inst, oi)
    assert sorted(int(k) for k in js["nuc"]) == sorted(oinfo.keys())
    for k, v in oinfo.items():
        j = js["nuc"][str(k)]
        assert j["bbox"] == v["bbox"].tolist() and j["centroid"] == v["centroid"].tolist()
        assert j["contour"] == v["contour"].tolist() and j["type"] == v["type"] and j["type_prob"] == v["type_prob"]
    assert np.array_equal(mat["inst_uid"].ravel(), np.array(sorted(oinfo.keys())))
    mgr.net.ctx.close()


@pytest.mark.gpu
def test_config0_single_270_tile_original_seg_only():
    """BASELINE configs[0]: one 270x270x3 tile, seg-only, `original` mode: U1 (one network patch) and
    U2 (tile-driver semantics: 4x4 patches of 270 stitched to 320^2, cropped to 270^2) vs the CPU oracle."""
    import torch
    from hover_net_b200 import synth
    from hover_net_b200.infer.tile import InferManager
    from oracle import hovernet_torch as O
    from oracle import postproc_oracle as P

    mode, nt = "original", None
    sd = synth.make_state_dict(mode, nt, seed=0)
    img = synth.make_patches(1, 270, seed=77)[0]
    mgr = InferManager(method={"model_args": {"nr_types": nt, "mode": mode}, "model_path": sd}, type_info_path=None)
    mgr.patch_input_shape, mgr.patch_output_shape, mgr.batch_size = 270, 80, 16
    tsd = O.to_torch_state_dict(sd)
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    # U1: the tile itself is exactly one network patch
    out = mgr.run_step(img[None])
    ref = O.infer_step(img[None], tsd, mode, nt)
    assert out.shape == (1, 80, 80, 3) and np.abs(out - ref).max() <= 1e-4
    oi, _ = P.process(out[0], nr_types=None, return_centroids=True)
    gi, _ = mgr.post_proc_func(out[0], nr_types=None, return_centroids=True)
    assert np.array_equal(gi, oi)
    # U2: tile-driver semantics
    pred_map, pred_inst, info = mgr.infer_image(img)
    assert pred_map.shape == (270, 270, 3) and pred_inst.shape == (270, 270)
    padded, pinfo, _ = tile._prepare_patching(img, 270, 80, True)
    assert len(pinfo) == 16
    outs = O.infer_step(np.stack([padded[y:y + 270, x:x + 270] for y, x, _, _ in pinfo]), tsd, mode, nt)
    ref_map = tile._stitch(list(pinfo), list(outs), img.shape)
    assert np.abs(pred_map - ref_map).max() <= 1e-4
    oi, oinfo = P.process(pred_map, nr_types=None, return_centroids=True)
    assert np.array_equal(pred_inst, oi) and sorted(info.keys()) == sorted(oinfo.keys())
    for k in info:
        assert np.array_equal(info[k]["bbox"], oinfo[k]["bbox"]) and np.array_equal(info[k]["centroid"], oinfo[k]["centroid"])
        assert np.array_equal(info[k]["contour"], oinfo[k]["contour"]) and info[k]["type"] is None
    mgr.net.ctx.close()


@pytest.mark.gpu
def test_config3_4k_tile_single_gpu_properties():
    """BASELINE configs[3] on one GPU: a 4096x4096 synthetic image through the tile driver (25x25 = 625
    fast-mode patches, stitched 4100^2 -> 4096^2, ONE whole-map post-processing with its global min/max).
    The CNN oracle cannot run 625 patches in a test; the map-level checks are size-independent:
    oracle post-processing of the device-produced map is bit-identical, the run is reproducible, and
    the instance table is consistent with inst_map."""
    from hover_net_b200 import synth
    from hover_net_b200.infer.tile import InferManager
    from oracle import postproc_oracle as P

    mode, nt = "fast", 6
    base = synth.make_patches(4, 256, seed=90)
    rng = np.random.default_rng(4)
    rows = [np.concatenate([base[rng.integers(0, 4)] for _ in range(16)], 1) for _ in range(16)]
    img = np.concatenate(rows, 0)
    assert img.shape == (4096, 4096, 3)
    sd = synth.make_state_dict(mode, nt, seed=0)
    mgr = InferManager(method={"model_args": {"nr_types": nt, "mode": mode}, "model_path": sd}, type_info_path=None)
    mgr.patch_input_shape, mgr.patch_output_shape, mgr.batch_size = 256, 164, 125
    padded, pinfo, _ = tile._prepare_patching(img, 256, 164, True)
    assert len(pinfo) == 625
    pred_map, pred_inst, info = mgr.infer_image(img)
    assert pred_map.shape == (4096, 4096, 4) and pred_inst.shape == (4096, 4096)
    oi, otab = P.process_table(pred_map, nt)
    assert np.array_equal(pred_inst, oi), "%d px differ" % int((pred_inst != oi).sum())
    ids, counts = np.unique(pred_inst[pred_inst > 0], return_counts=True)
    assert np.array_equal(ids, otab[:, 0]) and np.array_equal(counts, otab[:, 5])
    assert set(info.keys()) <= set(int(i) for i in ids)  # dict drops only the <3-point contours
    _, pred_inst2, _ = mgr.infer_image(img)
    assert np.array_equal(pred_inst, pred_inst2)
    mgr.net.ctx.close()


def _two_rank_tile_worker(rank, world, port, out):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from hover_net_b200 import synth
    from hover_net_b200.infer.tile import InferManager
    mode, nt = "fast", 6
    base = synth.make_patches(6, 256, seed=70)
    img = np.concatenate([np.concatenate(list(base[r * 3:(r + 1) * 3]), 1) for r in range(2)], 0)[:500, :610].copy()
    mgr = InferManager(method={"model_args": {"nr_types": nt, "mode": mode, "device": rank},
                               "model_path": synth.make_state_dict(mode, nt, seed=0)}, type_info_path=None)
    mgr.patch_input_shape, mgr.patch_output_shape, mgr.batch_size = 256, 164, 4
    pred, inst, info = mgr.infer_image(img, all_ranks=True)       # patch grid sharded over the ranks + all_reduce
    one = mgr.net.ctx.infer_tile(img, 256, 4)                     # the same image on this rank alone
    ok = bool(np.array_equal(pred, one[0]) and np.array_equal(inst, one[1]) and len(info) > 0)
    flags = [None] * world
    dist.all_gather_object(flags, ok)
    if rank == 0:
        out.put((flags, int(inst.max()), len(info)))
    dist.barrier()
    mgr.net.ctx.close()
    dist.destroy_process_group()


@pytest.mark.gpu
def test_config3_tile_sharded_over_two_gpus_equals_single_gpu():
    """configs[3] plumbing on real devices: one image, patch grid split over 2 ranks, maps summed by one NCCL
    all_reduce (disjoint supports) == the single-GPU device path, bit for bit, on both ranks."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import socket
    import torch.multiprocessing as mp
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_two_rank_tile_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    flags, max_id, n_info = q.get(timeout=600)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert flags == [True, True] and max_id > 0 and n_info > 0


def test_writers_match_reference(tmp_path):
    """QuPath TSV and the typed overlay vs the reference's own writers (goldens: oracle/gen_golden_tile.py)."""
    g = np.load(os.path.join(GOLD, "writers_tile.npz"))
    img = np.random.default_rng(99).integers(0, 256, (120, 150, 3), dtype=np.uint8)
    type_info = {0: ("nolabe", (0, 0, 0)), 1: ("neopla", (255, 0, 0)), 2: ("inflam", (0, 255, 0)), 3: ("connec", (0, 0, 255))}
    info = {int(k): {"contour": g["contour"][i], "centroid": g["centroid"][i], "type": int(g["type"][i])}
            for i, k in enumerate(g["ids"])}
    p = str(tmp_path / "a.tsv")
    tile._to_qupath(p, [v["centroid"] for v in info.values()], [v["type"] for v in info.values()], type_info)
    assert open(p).read() == str(g["tsv"])
    over = tile._overlay(img, info, draw_dot=True, type_colour=type_info, line_thickness=2)
    assert np.array_equal(over, g["overlay"])
