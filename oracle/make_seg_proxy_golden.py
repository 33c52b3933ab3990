"""Generate tests/golden/seg_proxy_*.npz for the proxy segmentation decoder (--seg_proxy) from the UNMODIFIED reference's
own modules on the CPU, in float32 and float64 (TEST INFRASTRUCTURE; run in the build container:
``python -m oracle.make_seg_proxy_golden``).

The reference builds the second decoder (``Decoder(num_classes, pretrain, do_segmentation=True)``,
BP/Networks/ERFNet.py:109-161) but its ``ERFNet.Net`` never asks for it, so here the ``decoder`` of the reference's
``LSQ_layer.Net`` is replaced by that Decoder.  The joint loss is main.py's end-to-end loss (the per-lane
``backprojection_loss`` calls averaged over the lanes; with --clas ``loss * weight_fit + (line + horizon) *
weight_class``) plus ``weight_seg_proxy * nn.CrossEntropyLoss([1] + [weight_seg] * L)(output_seg, gt)`` on an in-range
label map.  Parameters come from oracle/inputs.py (the second decoder's from the same distributions under their own
seed), images and loss targets as make_golden.py draws them.

Stored per case: the reference's state_dict key list with shapes, sampled output_seg entries, beta, the joint loss and
the proxy term, and sampled gradients of every parameter (layers1.*, the encoder -- which receives both decoders'
gradients -- and the heads), each in float32 and float64.
"""
import json
import math
import os
import zlib

import numpy as np
import torch
import torch.nn as nn

from . import inputs
from . import reference_import as ri
from .make_golden import GOLDEN_DIR, N_ACT_SAMPLES, N_GRAD_SAMPLES, summarize

CASES = [
    # name, nclasses, order, mask_pct, clas, B
    ("seg_proxy_l2_d2", 2, 2, 0.3, False, 2),
    ("seg_proxy_l4_d3_clas", 4, 3, 0.2, True, 2),
]
WEIGHT_SEG_PROXY = 0.5
PARAM_SEED, IMAGE_SEED, TARGET_SEED = 11, 3, 5


def branch_params(sd, seed):
    """Synthetic parameters for the keys of ``sd`` under net.decoder.layers1 (make_erfnet_params' distributions)."""
    rng = np.random.default_rng(seed)
    out = {}
    for k, v in sd.items():
        if not k.startswith("net.decoder.layers1.") or not (k.endswith(".weight") or k.endswith(".bias")):
            continue
        shape = tuple(v.shape)
        if len(shape) == 4:
            w = rng.standard_normal(shape) * math.sqrt(2.0 / (shape[1] * shape[2] * shape[3]))
        elif ".bn" in k and k.endswith(".weight"):
            w = 1.0 + 0.02 * rng.standard_normal(shape)
        else:
            w = 0.05 * rng.standard_normal(shape)
        out[k] = w.astype(np.float32)
    return out


def case_params(sd, L, clas):
    """Every parameter of the case, keyed like the reference's state_dict."""
    P = inputs.make_erfnet_params(3, L, seed=PARAM_SEED)
    P.update(branch_params(sd, PARAM_SEED + 1))
    if clas:
        for prefix, kind, seed in (("line_classification.", "line", 21), ("horizon_estimation.", "horizon", 22)):
            P.update({prefix + k: v for k, v in inputs.make_head_params(kind, seed).items()})
    return P


def case_targets(B, L, H, W, resize, seed):
    """label map [B, H, W] int64 in [0, L] (mostly background), gt_line [B, 4] and gt_horizon [B, resize] in {0, 1}."""
    rng = np.random.default_rng(seed)
    p = np.array([0.6] + [0.4 / L] * L)
    gt = rng.choice(L + 1, size=(B, H, W), p=p).astype(np.int64)
    gt_line = rng.integers(0, 2, size=(B, 4)).astype(np.float32)
    gt_horizon = rng.integers(0, 2, size=(B, resize)).astype(np.float32)
    return gt, gt_line, gt_horizon


def run_case(case):
    name, L, order, mask_pct, clas, B = case
    ns = ri.import_reference("Backprojection_Loss")
    H, W = 256, 512
    args = ri.make_args(ns, ["--nclasses", str(L), "--order", str(order), "--batch_size", str(B),
                             "--mask_percentage", str(mask_pct), "--end_to_end", "True", "--loss_policy", "backproject",
                             "--clas", str(int(clas))])
    torch.manual_seed(0)
    m = ns.LSQ_layer.Net(args)
    m.net.decoder = ns.ERFNet.Decoder(L, False, do_segmentation=True)
    sd = m.state_dict()
    P = case_params(sd, L, clas)
    missing = [k for k in sd if k not in P and not k.split(".")[-1] in ("running_mean", "running_var", "num_batches_tracked")]
    assert not missing, missing
    for k, v in P.items():
        assert tuple(sd[k].shape) == v.shape, (k, sd[k].shape, v.shape)
        sd[k] = torch.from_numpy(v)
    m.load_state_dict(sd)
    for mod in m.modules():
        if hasattr(mod, "dropout"):
            mod.dropout.p = 0
    m.train()
    x_np = inputs.make_images(B, H, W, seed=IMAGE_SEED)
    xgt_np, valid_np = inputs.make_loss_targets(B, 4, seed=TARGET_SEED)
    tseed = zlib.crc32(name.encode()) % 100000
    gt_np, line_np, hor_np = case_targets(B, L, H, W, args.resize, tseed)
    out = {"meta": json.dumps(dict(name=name, L=L, order=order, mask_pct=mask_pct, clas=clas, B=B, H=H, W=W,
                                   param_seed=PARAM_SEED, image_seed=IMAGE_SEED, target_seed=TARGET_SEED,
                                   label_seed=tseed, weight_seg=args.weight_seg, weight_seg_proxy=WEIGHT_SEG_PROXY,
                                   weight_fit=args.weight_fit, weight_class=args.weight_class)),
           "input_sha": inputs.sha256_of(x_np, xgt_np, valid_np, gt_np, line_np, hor_np),
           "param_sha": inputs.sha256_of(*[P[k] for k in sorted(P)]),
           "state_dict_keys": json.dumps([(k, list(v.shape)) for k, v in m.state_dict().items()]),
           "gt": gt_np.astype(np.uint8), "gt_line": line_np, "gt_horizon": hor_np}
    crit = ns.Loss_crit.backprojection_loss(args)
    for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
        if dt == torch.float64:
            m = m.double()
            m.grid = m.grid.double()
            m.ls_layer.tensor_ones = m.ls_layer.tensor_ones.double()
            m.ls_layer.reg_ls = m.ls_layer.reg_ls.double()
            for mod in m.modules():
                if isinstance(mod, torch.nn.BatchNorm2d):
                    mod.reset_running_stats()
        m.zero_grad()
        x = torch.from_numpy(x_np).to(dt)
        gt = torch.from_numpy(gt_np)
        res = m(x, torch.from_numpy(line_np), True, gt=gt)
        betas = [b for b in res[:4] if b is not None]
        line, horizon, output_seg = res[6], res[7], res[8]
        xgt, valid = torch.from_numpy(xgt_np), torch.from_numpy(valid_np)
        loss = 0
        for l in range(L):
            loss = loss + crit(betas[l], xgt[:, l], valid[:, l])[0]
        loss = loss / L
        if clas:
            loss_horizon = nn.BCEWithLogitsLoss()(horizon, torch.from_numpy(hor_np).to(dt)).double()
            loss_line = nn.BCEWithLogitsLoss()(line, torch.from_numpy(line_np).to(dt)).double()
            loss = loss * args.weight_fit + (loss_line + loss_horizon) * args.weight_class
        weights = torch.Tensor([1] + [args.weight_seg] * L).to(dt)
        ce = nn.CrossEntropyLoss(weights)(output_seg, gt)
        total = loss.double() + WEIGHT_SEG_PROXY * ce.double()
        total.backward()
        out["loss_" + tag] = np.array(float(total))
        out["ce_" + tag] = np.array(float(ce))
        out["beta_" + tag] = torch.stack([b.squeeze(-1) for b in betas], 1).detach().double().numpy()
        summarize("act_%s/output_seg" % tag, output_seg, N_ACT_SAMPLES, out)
        for n, p in m.named_parameters():
            if p.grad is not None:
                summarize("grad_%s/%s" % (tag, n), p.grad, N_GRAD_SAMPLES, out)
    out["params_without_grad"] = json.dumps([n for n, p in m.named_parameters() if p.grad is None])
    return name, out


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    for case in CASES:
        name, out = run_case(case)
        path = os.path.join(GOLDEN_DIR, name + ".npz")
        np.savez_compressed(path, **out)
        print(name, "loss f64 %.12g f32 %.12g  ce f64 %.12g  %d bytes" % (out["loss_f64"], out["loss_f32"], out["ce_f64"],
                                                                        os.path.getsize(path)))


if __name__ == "__main__":
    main()
