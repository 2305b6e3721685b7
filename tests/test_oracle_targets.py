"""CPU checks of the training targets and validation statistics: the numpy oracle of the device HV targets against
the reference's outcomes (tests/golden/targets_cases.npz), the `proc_valid_step_output` mirror against the
reference's scalars (tests/golden/valid_scalars.npz), `FileLoader`'s crops and the `run_valid` options."""
import json
import os

import numpy as np
import pytest

from oracle import targets_oracle as O
from oracle.gen_golden_targets import VALID_CASES, _raw

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cases():
    g = np.load(os.path.join(GOLDEN, "targets_cases.npz"))
    return g, json.loads(str(g["results"]))


def test_oracle_matches_reference_hv_maps():
    g, res = _cases()
    assert len(res) == 21
    for k, rec in enumerate(res):
        ann, crop = g["ann_%d" % k], tuple(int(v) for v in g["crop_%d" % k])
        hv, flags = O.hv_map(ann, crop)
        if "raises" in rec:
            assert rec["raises"] == "ValueError", rec
            assert flags != 0, rec["name"]
            continue
        assert flags == 0, rec["name"]
        assert hv.dtype == np.float32 and hv.tobytes() == g["hv_%d" % k].tobytes(), rec["name"]


def test_oracle_flag_kinds():
    g, res = _cases()
    by_name = {r["name"]: k for k, r in enumerate(res)}
    expect = {"wrap_nan": O.EMPTY_BOX, "no_background": O.NO_BACKGROUND | O.NO_BACKGROUND_CROP,
              "no_background_crop": O.NO_BACKGROUND_CROP}
    for name, bits in expect.items():
        k = by_name[name]
        assert O.hv_map(g["ann_%d" % k], tuple(g["crop_%d" % k]))[1] == bits, name


def test_gen_targets_crops_like_reference():
    from hover_net_b200.models.hovernet.targets import cropping_center
    g, res = _cases()
    for k, rec in enumerate(res):
        if "raises" in rec:
            continue
        ann, crop = g["ann_%d" % k], tuple(int(v) for v in g["crop_%d" % k])
        hv, _ = O.hv_map(ann, crop)
        assert np.array_equal(cropping_center(hv, crop), g["tgt_hv_%d" % k]), rec["name"]
        np_map = cropping_center((ann > 0).astype(np.int32), crop)
        assert np_map.dtype == g["tgt_np_%d" % k].dtype and np.array_equal(np_map, g["tgt_np_%d" % k]), rec["name"]


def test_oracle_errors():
    a = np.zeros((40, 40), np.int32)
    a[5:10, 5:10] = -3
    with pytest.raises(ValueError, match="negative"):
        O.hv_map(a, (20, 20))
    a = np.zeros((40, 40), np.int32)
    a[5:10, 5:10] = 2 ** 31 - 1  # one component: max id + 1 > 2^31 - 1
    with pytest.raises(ValueError, match="2\\^31"):
        O.hv_map(a, (20, 20))
    a[5:10, 5:10] = 2 ** 31 - 2
    assert O.hv_map(a, (20, 20))[1] == 0


def test_proc_valid_step_output_matches_reference():
    from hover_net_b200.models.hovernet.run_desc import proc_valid_step_output
    res = json.loads(str(np.load(os.path.join(GOLDEN, "valid_scalars.npz"))["results"]))
    assert len(res) == len(VALID_CASES)
    for k, (n, hw, nt) in enumerate(VALID_CASES):
        assert res[k]["nr_types"] == nt
        out = proc_valid_step_output(_raw(n, hw, nt, k), nr_types=nt)
        assert out["image"] == {}
        got, want = out["scalar"], res[k]["scalar"]
        assert list(got) == list(want)
        for key, (value, tname) in want.items():
            assert float(got[key]) == value and type(got[key]).__name__ == tname, (k, key, got[key], value)


def _write_patches(d, n, size, with_type, seed=0):
    from hover_net_b200 import synth
    rng = np.random.default_rng(seed)
    paths = []
    for i in range(n):
        img = rng.integers(0, 256, (size, size, 3))
        inst = synth.synth_instances(size, size, seed=seed * 100 + i)
        chans = [img, inst[..., None]]
        if with_type:
            chans.append(np.where(inst > 0, inst % 5, 0)[..., None])
        p = os.path.join(str(d), "p%03d.npy" % i)
        np.save(p, np.concatenate(chans, -1).astype(np.float64))  # extract_patches.py stores a float stack
        paths.append(p)
    return paths


def test_file_loader_crops_and_splits(tmp_path):
    from hover_net_b200.dataloader.train_loader import FileLoader
    paths = _write_patches(tmp_path, 2, 300, True)
    seen = []

    def gen(inst, mask_shape, **kw):
        seen.append((inst.copy(), tuple(mask_shape), kw))
        return {"np_map": "n", "hv_map": "h"}

    fl = FileLoader(paths, with_type=True, input_shape=[270, 270], mask_shape=[80, 80], mode="valid",
                    target_gen=(gen, {"k": 1}))
    assert len(fl) == 2
    d = fl[1]
    data = np.load(paths[1])
    img = data[15:285, 15:285, :3].astype(np.uint8)
    assert d["img"].dtype == np.uint8 and np.array_equal(d["img"], img)
    inst = data[15:285, 15:285, 3].astype(np.int32)
    assert np.array_equal(seen[0][0], inst) and seen[0][1:] == ((80, 80), {"k": 1})
    assert np.array_equal(d["tp_map"], data[15:285, 15:285, 4].astype(np.int32)[95:175, 95:175])
    assert d["np_map"] == "n" and d["hv_map"] == "h"
    fl = FileLoader(paths, with_type=False, input_shape=[256, 256], mask_shape=[164, 164], mode="valid",
                    target_gen=(gen, {}))
    assert "tp_map" not in fl[0] and np.array_equal(fl[0]["img"], np.load(paths[0])[22:278, 22:278, :3])
    with pytest.raises(NotImplementedError):
        FileLoader(paths, input_shape=[270, 270], mask_shape=[80, 80], mode="train", target_gen=(gen, {}))


def test_run_valid_arguments(tmp_path):
    from hover_net_b200 import run_valid
    a = run_valid.parse_args(["--model_path", "m.tar", "--valid_dir", "a", "--valid_dir", "b", "--nr_types", "6",
                              "--model_mode", "fast", "--batch_size", "8", "--precision", "high", "--json", "o.json"])
    assert (a.model_path, a.valid_dir, a.nr_types, a.model_mode, a.batch_size, a.precision, a.json) == \
        ("m.tar", ["a", "b"], 6, "fast", 8, "high", "o.json")
    a = run_valid.parse_args(["--model_path", "m", "--valid_dir", "a"])
    assert (a.model_mode, a.nr_types, a.precision, a.json) == ("original", 0, "highest", None)
    assert run_valid.SHAPES == {"original": ([270, 270], [80, 80]), "fast": ([256, 256], [164, 164])}
    with pytest.raises(SystemExit):
        run_valid.parse_args(["--model_path", "m", "--valid_dir", "a", "--precision", "medium"])
    for sub in ("b", "a"):
        os.makedirs(tmp_path / sub)
        for name in ("2.npy", "1.npy", "x.txt"):
            (tmp_path / sub / name).write_bytes(b"")
    got = run_valid.file_list([str(tmp_path / "b"), str(tmp_path / "a")])
    assert got == sorted(str(tmp_path / s / f) for s in "ab" for f in ("1.npy", "2.npy"))
