"""Test-time augmentation without a GPU: the view / bring-back table on analytic offset fields, the command-line
plumbing, and argument validation before any device call."""
import inspect

import numpy as np
import pytest

from hover_net_b200 import _lib, run_infer, run_valid

import tta_ref

BASE_ARGS = ["--model_mode=fast", "--nr_types=6", "--model_path=ck.tar"]
TILE_ARGS = ["tile", "--input_dir=in/", "--output_dir=out/"]


def _blob_field(mask):
    """[H,W,3] map of one blob: channel 0 the mask, then its HV offsets (x - cx, y - cy) inside the blob, 0 outside.
    The centroid comes from integer sums over a point-symmetric blob, so it is an exact integer in every frame."""
    ys, xs = np.nonzero(mask)
    cy, cx = ys.sum() // ys.size, xs.sum() // xs.size
    assert ys.sum() == cy * ys.size and xs.sum() == cx * xs.size
    yy, xx = np.mgrid[: mask.shape[0], : mask.shape[1]]
    out = np.zeros(mask.shape + (3,), np.float32)
    out[..., 0] = mask
    out[..., 1] = np.where(mask, xx - cx, 0)
    out[..., 2] = np.where(mask, yy - cy, 0)
    return out


def _ellipse(n, cy, cx, ry, rx):
    yy, xx = np.mgrid[:n, :n]
    return ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1.0


@pytest.mark.parametrize("n", [80, 81, 164, 165])
def test_every_view_comes_back_exactly(n):
    """The output a perfectly equivariant network gives on view t (the field of the viewed blob, computed in the view's
    own frame) is brought back to the input's field exactly, HV vectors included."""
    rng = np.random.default_rng(n)
    for cy, cx, ry, rx in ((n // 3, n // 2 + 7, 6.5, 11.5), (n - 15, 12, 9.5, 4.5)):
        mask = _ellipse(n, cy, cx, ry, rx)  # axis-aligned ellipse, off-centre, not symmetric under 90 degree turns
        truth = _blob_field(mask)
        seen = set()
        for t in range(tta_ref.NVIEWS):
            vm = tta_ref.view(mask[..., None], t)[..., 0]
            seen.add(vm.tobytes())
            back = tta_ref.unview(_blob_field(vm), t)
            assert np.array_equal(back, truth), (n, t)
        assert len(seen) == 8, "the eight views must be distinct"
        assert np.array_equal(tta_ref.merge([_blob_field(tta_ref.view(mask[..., None], t)[..., 0]) for t in range(8)]),
                              truth)
    z = rng.standard_normal((2, n, n, 4)).astype(np.float32)
    for t in range(tta_ref.NVIEWS):  # spatial inverse on arbitrary data, batch axis in front
        assert np.array_equal(tta_ref.unview(tta_ref.view(z, t), t, vector=False), z)


def test_view_table_matches_the_definition():
    """V_t(x) = np.rot90(np.flip(x, 1) if f else x, k, axes=(0, 1)) on an HWC patch; views() orders slot 8i + t."""
    x = np.arange(2 * 5 * 5 * 3, dtype=np.uint8).reshape(2, 5, 5, 3)
    v = tta_ref.views(x)
    assert v.shape == (16, 5, 5, 3)
    for i in range(2):
        for t in range(8):
            k, f = t % 4, t // 4
            assert np.array_equal(v[8 * i + t], np.rot90(np.flip(x[i], 1) if f else x[i], k, axes=(0, 1)))


def test_cli_tta_reaches_model_args_only_when_given():
    _, margs, _, _ = run_infer.parse(BASE_ARGS + ["--tta"] + TILE_ARGS)
    assert margs["method"]["model_args"] == {"nr_types": 6, "mode": "fast", "tta": True}
    _, margs, _, _ = run_infer.parse(BASE_ARGS + ["--tta", "--precision=high", "wsi", "--input_dir=a", "--output_dir=b"])
    assert margs["method"]["model_args"]["tta"] is True and margs["method"]["model_args"]["precision"] == "high"
    _, margs, _, _ = run_infer.parse(BASE_ARGS + TILE_ARGS)
    assert margs["method"]["model_args"] == {"nr_types": 6, "mode": "fast"}
    assert run_valid.parse_args(["--model_path=m", "--valid_dir=d", "--tta"]).tta is True
    assert run_valid.parse_args(["--model_path=m", "--valid_dir=d"]).tta is False


def test_default_tta_is_off():
    from hover_net_b200.models.hovernet import net_desc
    for fn in (net_desc.create_model, net_desc.HoVerNet.__init__, _lib.Context.__init__):
        assert inspect.signature(fn).parameters["tta"].default is False
    assert _lib.tta_code(False) == 0 and _lib.tta_code(True) == 1


def test_bad_tta_is_rejected_before_any_device_call(monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("libhvn was reached")

    monkeypatch.setattr(_lib, "lib", no_device)
    from hover_net_b200.models.hovernet.net_desc import create_model
    for bad in (1, 0, "yes", None, 8, np.bool_(True)):
        with pytest.raises(ValueError):
            create_model(mode="fast", nr_types=6, tta=bad)
        with pytest.raises(ValueError):
            _lib.Context(0, "fast", 6, tta=bad)
