"""Generate tests/golden/bev_clas.npz for the bird's-eye-view experiment's --clas heads and its validation score, from the
UNMODIFIED reference's own modules on the CPU (TEST INFRASTRUCTURE; run in the build container:
``python -m oracle.make_bev_clas_golden``).

  heads/<kind>/...   (a) the BEV Classification heads (Birds_Eye_View_Loss/Networks/LSQ_layer.py:170-228) on a seeded
                     encoder map, float32 and float64: out, sampled input and parameter gradients of sum(out * g),
                     running statistics (the layout of oracle/make_golden.py run_clas_heads)
  net/...            (b) a 4-lane BEV Net with --clas at B = 2, dropout-free: its state_dict keys and shapes, and in
                     float32 and float64 (net/f32/..., net/f64/...) beta, line, horizon and main.py:222-253's combined
                     loss with sampled parameter gradients
  score/...          (c) write_lsq_results(..., all_branches_ready=False, horizon_on=False) bytes and
                     LaneEval.bench_one_submit of seeded params over rows of Labels/Curve_parameters.json (48 and 56
                     h_samples), with and without no_ortho: absent lanes, curves that leave the image, a column beyond
                     int32.  Rows are stored as data (score/rows_jsonl).
"""
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch
import torch.nn as nn

from . import inputs
from . import reference_import as ri
from .make_golden import GOLDEN_DIR, summarize

MAP_SEED, G_SEEDS, PARAM_SEEDS = 21, {"line": 51, "horizon": 52}, {"line": 61, "horizon": 62}
NET_PARAM_SEED, NET_IMAGE_SEED, NET_TARGET_SEED = 11, 3, 5
SCORE_SEED = 7


def bev_head_params(kind, seed):
    """Parameters of one BEV head keyed like its state_dict: the BP head's distributions (oracle/inputs.py), the line
    head's last layer replaced by four Linear(128, 3)."""
    P = inputs.make_head_params(kind, seed)
    if kind == "line":
        del P["fully_connected_line1.weight"], P["fully_connected_line1.bias"]
        rng = np.random.default_rng(seed + 1000)
        for k in range(1, 5):
            P["fully_connected_line%d.weight" % k] = (rng.standard_normal((3, 128)) * np.sqrt(2.0 / 128)).astype(np.float32)
            P["fully_connected_line%d.bias" % k] = (0.05 * rng.standard_normal(3)).astype(np.float32)
    return P


def load(m, P):
    sd = m.state_dict()
    for k, v in P.items():
        assert tuple(sd[k].shape) == v.shape, (k, sd[k].shape, v.shape)
        sd[k] = torch.from_numpy(v)
    m.load_state_dict(sd)


def net_targets(B, resize, seed):
    """gt_line [B, 4] int64 in 0..2 and gt_horizon [B, resize] in {0, 1}, as the BEV loader forms them."""
    rng = np.random.default_rng(seed)
    return rng.integers(0, 3, size=(B, 4)).astype(np.int64), rng.integers(0, 2, size=(B, resize)).astype(np.float32)


def net_params(seed):
    """The lane-fit parameters of the --clas Net case: [B, 4, 3] float32, lane 3 of image 1 absent."""
    p = (np.random.default_rng(seed).normal(size=(2, 4, 3)) * np.array([0.1, 0.1, 0.3]) + np.array([0, 0, 0.5]))
    p = p.astype(np.float32)
    p[1, 3] = 0.0
    return p


def run_heads(ns, out):
    x_np = inputs.make_encoder_map(2, seed=MAP_SEED)
    for kind in ("line", "horizon"):
        P = bev_head_params(kind, PARAM_SEEDS[kind])
        for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
            torch.manual_seed(0)
            m = ns.LSQ_layer.Classification(kind, size=(32, 64), channels_in=128, resize=256)
            load(m, P)
            m = m.to(dt).train()
            x = torch.from_numpy(x_np).to(dt).requires_grad_(True)
            y = m(x)
            g = torch.from_numpy(np.random.default_rng(G_SEEDS[kind]).standard_normal(tuple(y.shape))).to(dt)
            (y * g).sum().backward()
            out["heads/%s/out_%s" % (kind, tag)] = y.detach().double().numpy()
            summarize("heads/%s/dx_%s" % (kind, tag), x.grad, 4096, out)
            for n, p in m.named_parameters():
                summarize("heads/%s/grad_%s/%s" % (kind, tag, n), p.grad, 1024, out)
            for n, b in m.named_buffers():
                if n.endswith("running_mean") or n.endswith("running_var"):
                    out["heads/%s/buf_%s/%s" % (kind, tag, n)] = b.detach().double().numpy()
        out["heads/%s/g" % kind] = np.random.default_rng(G_SEEDS[kind]).standard_normal(tuple(y.shape))


def net_grad_sampled(name):
    """The parameters whose gradients (b) samples: both heads, and the encoder's first and the decoder's last layer."""
    return name.startswith(("line_classification.", "horizon_estimation.", "net.encoder.initial_block",
                            "net.decoder.output_conv"))


def run_net(ns, out):
    B = 2
    args = ri.make_args(ns, ["--nclasses", "4", "--order", "2", "--batch_size", str(B), "--loss_policy", "area",
                             "--clas", "True"])
    torch.manual_seed(0)
    model = ns.LSQ_layer.Net(args)
    sd = model.state_dict()
    out["net/keys"] = np.array(json.dumps([[k, list(v.shape)] for k, v in sd.items()]))
    load(model, {k: v for k, v in net_all_params().items() if k in sd})
    for mod in model.modules():
        if hasattr(mod, "dropout"):
            mod.dropout.p = 0            # dropout-free, as the other network fixtures
    model.train()
    x_np = inputs.make_images(B, 256, 512, seed=NET_IMAGE_SEED)
    gt_line, gt_horizon = net_targets(B, 256, NET_TARGET_SEED)
    params_np = net_params(NET_TARGET_SEED)
    for tag, dt in (("f32", torch.float32), ("f64", torch.float64)):
        if dt == torch.float64:
            model = model.double()
            model.M = model.M.double()
            model.project_layer.base_grid = model.project_layer.base_grid.double()
            model.ls_layer.tensor_ones = model.ls_layer.tensor_ones.double()
            model.ls_layer.reg_ls = model.ls_layer.reg_ls.double()
        model.zero_grad()
        params = torch.from_numpy(params_np).to(dt)
        beta0, beta1, beta2, beta3, _, _, _, line, horizon = model(torch.from_numpy(x_np).to(dt), True)
        crit = ns.Loss_crit.Area_Loss(args.order, args.weight_funct)
        gt0, gt1, gt2, gt3 = params[:, 0, :], params[:, 1, :], params[:, 2, :], params[:, 3, :]
        loss = crit(beta0, gt0) + crit(beta1, gt1)                                 # BEV/main.py:222-237
        mask_llhs = torch.prod(gt2 != 0, 1).unsqueeze(1).unsqueeze(1).expand_as(beta2).type(torch.FloatTensor)
        mask_rrhs = torch.prod(gt3 != 0, 1).unsqueeze(1).unsqueeze(1).expand_as(beta3).type(torch.FloatTensor)
        loss += crit(beta2 * mask_llhs.to(dt), gt2) + crit(beta3 * mask_rrhs.to(dt), gt3)
        loss_horizon = nn.BCEWithLogitsLoss()(horizon, torch.from_numpy(gt_horizon).to(dt))  # :246-253
        loss_line = nn.CrossEntropyLoss()(line, torch.from_numpy(gt_line))
        loss = loss * args.weight_fit + (loss_line + loss_horizon) * args.weight_class
        loss.backward()
        pre = "net/%s/" % tag
        out[pre + "beta"] = torch.cat((beta0, beta1, beta2, beta3), 2).transpose(1, 2).detach().double().numpy()
        out[pre + "line"] = line.detach().double().numpy()
        out[pre + "horizon"] = horizon.detach().double().numpy()
        out[pre + "loss"] = np.array(float(loss.detach()))
        for n, p in model.named_parameters():
            if p.grad is not None and net_grad_sampled(n):
                summarize(pre + "grad/" + n, p.grad, 256, out)


def net_all_params():
    """Every parameter of the (b) case keyed like the BEV Net's state_dict (ERFNet and both heads)."""
    P = inputs.make_erfnet_params(3, 4, seed=NET_PARAM_SEED)
    for prefix, kind in (("line_classification.", "line"), ("horizon_estimation.", "horizon")):
        P.update({prefix + k: v for k, v in bev_head_params(kind, PARAM_SEEDS[kind] + 100).items()})
    return P


def load_lane_eval():
    """The reference BEV LaneEval class, imported unmodified; its `import ujson as json` gets the standard json module."""
    import importlib.util
    sys.modules.setdefault("ujson", types.SimpleNamespace(loads=json.loads, dumps=json.dumps))
    spec = importlib.util.spec_from_file_location("_ref_bev_eval_lane",
                                                  os.path.join(ri.REFERENCE_ROOT, "Birds_Eye_View_Loss", "eval_lane.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.LaneEval


def score_rows():
    """12 rows of Labels/Curve_parameters.json, 6 with 48 and 6 with 56 h_samples; row 2's lane 1 and row 7's lane 3
    made absent (all -2)."""
    path = os.path.join(ri.REFERENCE_ROOT, "Birds_Eye_View_Loss", "Labels", "Curve_parameters.json")
    rows = [json.loads(line) for line in open(path).readlines()]
    pick = [r for r in rows if len(r["h_samples"]) == 48][:6] + [r for r in rows if len(r["h_samples"]) == 56][:6]
    pick[2]["lanes"][1] = [-2] * len(pick[2]["h_samples"])
    pick[7]["lanes"][3] = [-2] * len(pick[7]["h_samples"])
    return pick


def score_params(rows, seed):
    """[N, 4, 3] float32 fitted curves: each row's poly_params with noise (most lanes near their labels), two lanes that
    leave the image, one whose columns exceed int32."""
    rng = np.random.default_rng(seed)
    p = np.array([r["poly_params"] for r in rows], np.float64)
    p = p + rng.normal(size=p.shape) * np.array([2e-4, 5e-3, 5e-3])
    p[3, 0] = [0.0, 0.0, -3.0]                   # left of the image
    p[9, 2] = [40.0, -20.0, 3.0]                 # far outside on one side
    p[5, 1] = [0.0, 0.0, 3.0e7]                  # x * 1279 beyond int32 inside the labelled rows
    return p.astype(np.float32)


def run_score(out):
    mod = sys.modules.get("_ref_bev_load_data_new")
    if mod is None:
        from .make_loader_bev_golden import load_reference
        mod = load_reference()
    LaneEval = load_lane_eval()
    rows = score_rows()
    params = score_params(rows, SCORE_SEED)
    out["score/rows_jsonl"] = np.frombuffer("".join(json.dumps(r) + "\n" for r in rows).encode(), np.uint8)
    out["score/params"] = params
    with tempfile.TemporaryDirectory() as tmp:
        src = os.path.join(tmp, "validation_set_dst.json")
        with open(src, "w") as f:
            for r, p in zip(rows, params):
                r = dict(r)
                r["params"] = p.tolist()
                r["line_id"] = [1, 1, 1, 1]
                r["horizon_est"] = [0.0] * 256
                json.dump(r, f)
                f.write("\n")
        out["score/dst_bytes"] = np.frombuffer(open(src, "rb").read(), np.uint8)
        for no_ortho in (False, True):
            dst = os.path.join(tmp, "ls_result.json")
            mod.write_lsq_results(src, dst, 4, False, False, 256, no_ortho=no_ortho)
            tag = "score/no_ortho%d" % int(no_ortho)
            out[tag + "/ls_bytes"] = np.frombuffer(open(dst, "rb").read(), np.uint8)
            out[tag + "/file"] = np.asarray(LaneEval.bench_one_submit(dst, src), np.float64)
            preds = [json.loads(line) for line in open(dst).readlines()]
            out[tag + "/per_row"] = np.array([LaneEval.bench(q["lanes"], r["lanes"], r["h_samples"], 20)
                                              for q, r in zip(preds, rows)], np.float64)


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    out = {"meta": np.array(json.dumps(dict(B=2, map_seed=MAP_SEED, param_seeds=PARAM_SEEDS, g_seeds=G_SEEDS,
                                            net_param_seed=NET_PARAM_SEED, net_image_seed=NET_IMAGE_SEED,
                                            net_target_seed=NET_TARGET_SEED, score_seed=SCORE_SEED)))}
    orig = torch.masked_select
    # Area_Loss masks with a uint8 tensor, as torch 1.1 accepted (oracle/make_golden.py run_area_loss)
    torch.masked_select = lambda x, mask: orig(x, mask.bool() if mask.dtype == torch.uint8 else mask)
    try:
        ns = ri.import_reference("Birds_Eye_View_Loss")
        run_heads(ns, out)
        run_net(ns, out)
    finally:
        torch.masked_select = orig
        ri.purge()
    run_score(out)
    path = os.path.join(GOLDEN_DIR, "bev_clas.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")
    return 0


if __name__ == "__main__":
    sys.exit(main())
