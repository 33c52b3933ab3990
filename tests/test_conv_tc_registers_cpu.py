"""The TF32 and 3xTF32 instantiations of the 3-tap convolution kernel (csrc/conv_tc.cu) fit the 168-register cap of its
288-thread CTA without spilling: the epilogue operands it loads before the MMAs must stay in registers for their
latency to hide behind them.  Compiles for sm_90a with -Xptxas -v; no GPU needed."""
import os
import re
import shutil
import subprocess

import pytest

from lanedetection_end2end_b200.csrc import build as B

SRC = os.path.join(B.HERE, "conv_tc.cu")


def test_tf32_and_x3_conv_tc_kernels_do_not_spill(tmp_path):
    if not (os.path.exists(B.NVCC) or shutil.which(B.NVCC)):
        pytest.skip("nvcc not found")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", SRC, "-o", str(tmp_path / "conv_tc.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    # ptxas: "Compiling entry function '<name>'", then "<n> bytes stack frame, <s> bytes spill stores, <l> bytes spill loads"
    found = {}
    name = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name:
            k = re.search(r"conv1d_tc_kernelILi(\d+)ELi(\d)ELb([01])ELb([01])E", name)
            if k:
                found[k.groups()] = (int(m.group(1)), int(m.group(2)))
            name = None
    # precision 0 = TF32, 1 = 3xTF32 (tc_ptx.cuh TcPrec); C in {64, 128}, resident or streamed weights, fp32 activations
    want = [(c, p, res, "0") for c in ("64", "128") for p in ("0", "1") for res in ("0", "1")]
    for key in want:
        assert key in found, (key, sorted(found))
        assert found[key] == (0, 0), ("C, precision, resident weights, bf16 input", key, "spill stores / loads", found[key])
