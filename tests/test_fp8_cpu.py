"""The inference-only fp8 convolution mode without a GPU:
  * accuracy of the mode's arithmetic (oracle/fp8_oracle.py) on the golden inputs, in eval mode with running statistics
    from one training-mode forward: beta's norm-wise error from the fp64 eval forward of the same model (printed; the
    GPU test compares the H100 against the same emulation);
  * the fp8 instantiations of the 3-tap kernel compile for sm_90a within the 168-register cap without spilling;
  * with the mode set, Net refuses a training forward and a grad-enabled forward;
  * a mode switch never serves another mode's cached operands (ops_eval's per-module cache)."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from oracle import fp8_oracle as fo


@pytest.mark.parametrize("name", ["net_l2_d2", "net_l4_d3"])
def test_fp8_eval_emulation_accuracy(name):
    rec = fo.emulate_golden_case(name)[0]
    print(rec)
    assert rec["beta_normwise_err_fp8"] < 3e-2, rec
    assert rec["beta_normwise_err_fp8"] > rec["beta_normwise_err_bf16"] > rec["beta_normwise_err_fp32"], rec


def test_fp8_conv_tc_kernels_do_not_spill(tmp_path):
    from lanedetection_end2end_b200.csrc import build as B
    if not (os.path.exists(B.NVCC) or shutil.which(B.NVCC)):
        pytest.skip("nvcc not found")
    r = subprocess.run([B.NVCC] + B.FLAGS + ["-Xptxas", "-v", "-c", os.path.join(B.HERE, "conv_tc.cu"), "-o",
                        str(tmp_path / "conv_tc.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    # ptxas: "Compiling entry function '<name>'", then the stack / spill line, then "Used <r> registers"
    found, name, spills = {}, None, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            name, spills = m.group(1), None
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            spills = (int(m.group(1)), int(m.group(2)))
            continue
        m = re.search(r"Used (\d+) registers", line)
        if m and name:
            k = re.search(r"conv1d_tc_kernelILi(\d+)ELi3ELb([01])ELb([01])E", name)   # precision 3 = FP8 (TcPrec)
            if k:
                found[k.groups()] = (spills, int(m.group(1)))
            name = None
    # C in {64, 128}, resident or streamed weights, fp32 or bf16 activations
    for key in [(c, res, abf) for c in ("64", "128") for res in ("0", "1") for abf in ("0", "1")]:
        assert key in found, (key, sorted(found))
        assert found[key][0] == (0, 0) and found[key][1] <= 168, ("C, resident weights, bf16 input", key, found[key])


def _small_net():
    from lanedetection_end2end_b200.Networks.ERFNet import Net
    return Net(in_channels=3, out_channels=2)


def test_fp8_mode_refuses_training_and_autograd_forwards():
    from lanedetection_end2end_b200 import ops_net
    net = _small_net()
    x = torch.zeros(1, 3, 32, 64)
    ops_net.set_conv_mode("fp8")
    with pytest.raises(RuntimeError, match="inference-only"):
        net.train()(x, True)
    with pytest.raises(RuntimeError, match="inference-only"):
        net.eval()(x, True)                       # grad mode on, parameters require grad: would build a graph
    with pytest.raises(RuntimeError, match="inference-only"):
        net.eval()(x.requires_grad_(), True)
    # the blocks refuse on their own too
    blk = net.encoder.layers[1].train()
    with pytest.raises(RuntimeError, match="inference-only"):
        blk(torch.zeros(1, 64, 8, 16).to(memory_format=torch.channels_last))
    # and the mode is a real mode
    ops_net.set_conv_mode("tf32x3")
    with pytest.raises(ValueError):
        ops_net.set_conv_mode("fp4")


def test_mode_switch_never_serves_another_modes_cached_operands():
    from lanedetection_end2end_b200 import ops_eval, ops_net
    from lanedetection_end2end_b200.Networks.ERFNet import non_bottleneck_1d
    torch.manual_seed(0)
    blk = non_bottleneck_1d(64, 0.0, 2).eval()
    for bn in (blk.bn1, blk.bn2):
        bn.running_mean.uniform_(-0.5, 0.5)
        bn.running_var.uniform_(0.5, 2.0)

    def ops(mode):
        ops_net.set_conv_mode(mode)
        return ops_eval.nb1d_operands(blk, False)

    bf = ops("bf16")
    assert [t[0].dtype for t in bf] == [torch.bfloat16] * 2
    f8 = ops("fp8")
    assert len(f8) == 4 and all(t[0].dtype == torch.uint8 and t[0].shape == (64, 192) for t in f8)
    # the operands are the oracle's quantisation of the weights, in the packed layout
    w1 = blk.conv3x1_1.weight.detach()
    q, s = fo.quantize_weight(w1)
    assert torch.equal(f8[0][1], s)
    assert torch.equal(f8[0][0].view(torch.float8_e4m3fn).float(), q.permute(0, 2, 3, 1).reshape(64, 192))
    x3 = ops("tf32x3")
    assert [t[0].dtype for t in x3] == [torch.float32] * 2 and x3[0][0].shape == (2, 64, 192)
    bf2 = ops("bf16")
    assert all(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) for a, b in zip(bf, bf2))
    assert ops("fp8")[0][0].dtype == torch.uint8
    # a parameter update rebuilds the fp8 operands as well
    with torch.no_grad():
        blk.conv3x1_1.weight.mul_(2.0)
    assert torch.equal(ops("fp8")[0][1], 2 * s)
