"""Precision option without a GPU: CLI plumbing, argument validation, and the sm_90a compile of the single-product
kernel variants."""
import inspect
import os
import re
import shutil
import subprocess

import pytest

from hover_net_b200 import _lib, run_infer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_ARGS = ["--model_mode=fast", "--nr_types=6", "--model_path=ck.tar"]
TILE_ARGS = ["tile", "--input_dir=in/", "--output_dir=out/"]


def test_cli_precision_reaches_model_args():
    _, margs, _, _ = run_infer.parse(BASE_ARGS + ["--precision=high"] + TILE_ARGS)
    assert margs["method"]["model_args"] == {"nr_types": 6, "mode": "fast", "precision": "high"}
    _, margs, _, _ = run_infer.parse(BASE_ARGS + ["--precision", "high", "wsi", "--input_dir=a", "--output_dir=b"])
    assert margs["method"]["model_args"]["precision"] == "high"


def test_default_precision_is_highest():
    _, margs, _, _ = run_infer.parse(BASE_ARGS + TILE_ARGS)
    assert margs["method"]["model_args"].get("precision", "highest") == "highest"
    _, margs, _, _ = run_infer.parse(BASE_ARGS + ["--precision=highest"] + TILE_ARGS)
    assert margs["method"]["model_args"].get("precision", "highest") == "highest"
    from hover_net_b200.models.hovernet import net_desc
    for fn in (net_desc.create_model, net_desc.HoVerNet.__init__, _lib.Context.__init__):
        assert inspect.signature(fn).parameters["precision"].default == "highest"
    assert _lib.precision_code("highest") == 0 and _lib.precision_code("high") == 1


def test_bad_precision_is_rejected_before_any_device_call(monkeypatch):
    with pytest.raises(SystemExit):
        run_infer.parse(BASE_ARGS + ["--precision=bogus"] + TILE_ARGS)

    def no_device(*a, **k):
        raise AssertionError("libhvn was reached")

    monkeypatch.setattr(_lib, "lib", no_device)
    from hover_net_b200.models.hovernet.net_desc import create_model
    for bad in ("bogus", "medium", None, 1):
        with pytest.raises(ValueError):
            create_model(mode="fast", nr_types=6, precision=bad)
        with pytest.raises(ValueError):
            _lib.Context(0, "fast", 6, precision=bad)


def _ptxas_report(src):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not (os.path.exists(nvcc) or shutil.which(nvcc)):
        pytest.skip("nvcc not available")
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                            "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", src, "-o", os.path.join(d, "k.o")],
                           capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    out, kernels, name = r.stdout + r.stderr, {}, None
    for line in out.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            kernels.setdefault(name, {})["spill"] = int(m.group(1)) + int(m.group(2))
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            kernels.setdefault(name, {})["regs"] = int(m.group(1))
    return kernels


def test_single_product_kernels_compile_for_sm90a():
    """Every single-product (precision "high") instantiation of k_conv_tc is built for sm_90a without spills, beside
    the unchanged two-plane ones; the single-product stem is built too."""
    k = _ptxas_report(os.path.join(ROOT, "hover_net_b200", "csrc", "conv_tc.cu"))
    # mangled template arguments: k_conv_tc<BLOCK_N, STAGES, MODE, XF, ONE>
    conv = {n: v for n, v in k.items() if "k_conv_tc" in n}
    single = [n for n in conv if "Lb1EEEv" in n]
    double = [n for n in conv if "Lb0EEEv" in n]
    assert len(single) == 13 and len(double) == 13, sorted(conv)
    for n in single + double:
        assert conv[n]["spill"] == 0, (n, conv[n])
        assert conv[n]["regs"] <= 168, (n, conv[n])  # 384 threads, one CTA per SM
    assert any("k_conv0_tcILb1E" in n for n in k) and any("k_conv0_tcILb0E" in n for n in k)
