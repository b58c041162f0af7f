"""The development benchmarks under tools/ start on a machine without a GPU, and take their measuring from
tools/measure.py rather than from private copies."""
import glob
import importlib.util
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, "tools")
# every benchmark on tools/measure.py; dp_timeline.py takes positional arguments and has no --help
SCRIPTS = ["cat_bench", "clip_bench", "conv_nd_bench", "criteria_bench", "cross_entropy_bench", "embedding_bench",
           "f32_conv_bench", "f32_gemm_bench", "gemm_sweep", "norm_bench", "optim_bench", "pool_bench", "rnn_bench"]


@pytest.mark.parametrize("name", SCRIPTS)
def test_help(name):
    r = subprocess.run([sys.executable, os.path.join(TOOLS, name + ".py"), "--help"], capture_output=True, text=True,
                       timeout=120)
    assert r.returncode == 0, r.stderr
    assert r.stdout.startswith("usage:")


def test_measure_imports():
    spec = importlib.util.spec_from_file_location("measure", os.path.join(TOOLS, "measure.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    for name in ("Clock", "setup", "window", "alternate", "capture", "kernel_ms"):
        assert callable(getattr(m, name)), name
    assert set(m.DATASHEET) == {"hbm_gbps", "bf16_tflops", "tf32_tflops", "fp32_tflops"}


def test_timing_lives_in_measure():
    private = re.compile(r"torch\.cuda\.Event\(|nvmlInit|nvidia-smi|\bHBM_\w+\s*=|from (cat_bench|gemm_sweep) import")
    found = [f"{os.path.basename(path)}:{i}" for path in sorted(glob.glob(os.path.join(TOOLS, "*.py")))
             if not path.endswith("measure.py")
             for i, line in enumerate(open(path), 1) if private.search(line)]
    assert not found, found
