"""The validation loss on the CPU: the float64 restatement (tests/loss_ref.py) and run_desc.loss_scalars against the
reference's own loss functions (tests/golden/loss_cases.npz, oracle/gen_golden_loss.py), the names and weights, and
the `run_valid --loss` command line."""
import json
import os

import numpy as np
import pytest

from hover_net_b200 import run_valid
from hover_net_b200.models.hovernet import run_desc

import loss_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "loss_cases.npz")


def golden_cases():
    g = np.load(GOLDEN)
    res = json.loads(str(g["results"]))
    for name, r in res.items():
        nt = r["nt"]
        yield name, g["probs_" + name], g["fg_" + name], g["hv_" + name], (g["tp_" + name] if nt else None), r


def test_restatement_matches_reference_golden():
    n = 0
    for name, probs, fg, hv, tp, want in golden_cases():
        got = run_desc.loss_scalars(loss_ref.sums(probs, fg, hv, tp), fg.size)
        assert list(got) == [k for k in want if k != "nt"], name
        for k, v in got.items():
            assert abs(v - want[k]) <= 1e-5 * abs(want[k]) + 1e-7, (name, k, v, want[k])
        n += 1
    assert n == 10


def test_golden_covers_the_edge_cases():
    cases = {name: (probs, fg, tp) for name, probs, fg, hv, tp, _ in golden_cases()}
    assert not cases["no_fg_t0"][1].any() and cases["all_fg_t5"][1].all()
    p = cases["clamp_t6"][0]
    assert set(np.unique(p[..., [0, 1, 4, 5, 6, 7, 8, 9]])) == {0.0, 1.0}
    p, _, tp = cases["absent_t6"]
    assert not p[..., 4 + 3].any() and not (tp == 3).any()
    shapes = {c[0].shape[:3] for c in cases.values()}
    assert (1, 80, 80) in shapes and (1, 164, 164) in shapes and (33, 7, 5) in shapes and (4, 3, 3) in shapes


def test_loss_scalars_names_and_weights():
    s = np.arange(1, 11, dtype=np.float64)
    got = run_desc.loss_scalars(s, 4)
    assert list(got) == ["loss_np_bce", "loss_np_dice", "loss_hv_mse", "loss_hv_msge", "overall_loss"]
    assert got["loss_np_bce"] == 1 / 4
    assert got["loss_np_dice"] == (1 - (2 * 2 + 1e-3) / (4 + 6 + 1e-3)) + (1 - (2 * 3 + 1e-3) / (5 + 7 + 1e-3))
    assert got["loss_hv_mse"] == 8 / 8
    assert got["loss_hv_msge"] == 9 / (2 * 10 + 1e-8)
    assert got["overall_loss"] == sum(v for k, v in got.items() if k != "overall_loss")
    nt = 5
    t = np.arange(1, 12 + 3 * nt, dtype=np.float64)
    got = run_desc.loss_scalars(t, 7)
    assert list(got) == ["loss_tp_bce", "loss_tp_dice", "loss_np_bce", "loss_np_dice", "loss_hv_mse",
                         "loss_hv_msge", "overall_loss"]
    assert got["loss_tp_bce"] == 11 / 7
    i, l, r = t[11:16], t[16:21], t[21:26]
    assert got["loss_tp_dice"] == float(np.sum(1.0 - (2.0 * i + 1e-3) / (l + r + 1e-3)))
    opts = {"np": {"bce": 2.0, "dice": 0.5}, "hv": {"msge": 3.0}, "tp": {"dice": 1.0}}
    w = run_desc.loss_scalars(t, 7, loss_opts=opts)
    assert list(w) == ["loss_tp_dice", "loss_np_bce", "loss_np_dice", "loss_hv_msge", "overall_loss"]
    assert w["overall_loss"] == (w["loss_tp_dice"] + 2.0 * w["loss_np_bce"] + 0.5 * w["loss_np_dice"]
                                 + 3.0 * w["loss_hv_msge"])
    assert run_desc.LOSS_OPTS == {"np": {"bce": 1, "dice": 1}, "hv": {"mse": 1, "msge": 1},
                                  "tp": {"bce": 1, "dice": 1}}


def test_set_loss_is_the_loss_of_the_concatenated_batch():
    name, probs, fg, hv, tp, _ = next(c for c in golden_cases() if c[0] == "c7x5_b33_t6")
    whole = run_desc.loss_scalars(loss_ref.sums(probs, fg, hv, tp), fg.size)
    parts = sum(loss_ref.sums(probs[a:a + 5], fg[a:a + 5], hv[a:a + 5], tp[a:a + 5]) for a in range(0, 33, 5))
    split = run_desc.loss_scalars(parts, fg.size)
    for k in whole:
        assert abs(whole[k] - split[k]) <= 1e-12 * abs(whole[k]) + 1e-15, k


class _FakeCtx:
    """Stands in for the device: `valid` / `valid_loss` return fixed counts and sums per batch."""
    nr_types = None

    def __init__(self):
        self.calls = []

    def out_shape(self, h, w):
        return 80, 80, 3

    def malloc_host(self, n):
        buf = np.zeros(n, np.uint8)
        self.__dict__.setdefault("_bufs", []).append(buf)
        return buf.ctypes.data

    def free_host(self, p):
        pass

    def valid(self, img, inst, typ):
        self.calls.append("valid")
        return np.array([100, 10, 30], np.int64), 2.5, np.zeros(len(img), np.int32)

    def valid_loss(self, img, inst, typ):
        self.calls.append("valid_loss")
        sums = np.arange(1, 11, dtype=np.float64) * len(img)
        return np.array([100, 10, 30], np.int64), 2.5, np.zeros(len(img), np.int32), sums, None


@pytest.fixture
def fake_run(tmp_path, monkeypatch):
    from hover_net_b200.dataloader import train_loader
    from hover_net_b200.models.hovernet import net_desc
    for i in range(3):
        np.save(tmp_path / ("p%d.npy" % i), np.zeros((2, 2, 4)))
    ctx = _FakeCtx()

    class Net:
        def __init__(self):
            self.ctx = ctx

        def load_state_dict(self, sd, strict=True):
            pass

    class Loader:
        def __init__(self, files, **kw):
            pass

        def load(self, i):
            return np.zeros((270, 270, 3), np.uint8), np.zeros((270, 270), np.int32), None

    monkeypatch.setattr(net_desc, "create_model", lambda **kw: Net())
    monkeypatch.setattr(train_loader, "FileLoader", Loader)
    ck = tmp_path / "ck.npz"
    np.savez(ck, a=np.zeros(1))
    base = ["--model_path", str(ck), "--valid_dir", str(tmp_path), "--batch_size", "2"]
    return ctx, base, tmp_path


def test_run_valid_loss_option(fake_run, capsys):
    ctx, base, tmp = fake_run
    assert run_valid.parse_args(base).loss is False
    assert run_valid.parse_args(base + ["--loss", "--tta", "--precision", "high"]).loss is True
    run_valid.main(base + ["--json", str(tmp / "plain.json")])
    plain_out = capsys.readouterr().out
    assert ctx.calls == ["valid", "valid"]
    plain = json.loads((tmp / "plain.json").read_text())
    assert list(plain) == ["np_acc", "np_dice", "hv_mse"]
    ctx.calls.clear()
    run_valid.main(base + ["--loss", "--json", str(tmp / "loss.json")])
    loss_out = capsys.readouterr().out
    assert ctx.calls == ["valid_loss", "valid_loss"]
    got = json.loads((tmp / "loss.json").read_text())
    names = ["loss_np_bce", "loss_np_dice", "loss_hv_mse", "loss_hv_msge", "overall_loss"]
    assert list(got) == list(plain) + names
    assert {k: got[k] for k in plain} == plain
    assert loss_out.startswith(plain_out)
    # three patches in batches of 2 and 1: the set's sums are 3 x (1..10)
    want = run_desc.loss_scalars(np.arange(1, 11, dtype=np.float64) * 3, 3 * 80 * 80)
    assert {k: got[k] for k in names} == want
    printed = dict(line.split(": ") for line in loss_out.strip().split("\n"))
    assert {k: float(v) for k, v in printed.items()} == got
