"""The fused optimizer update (csrc/optim.cu, optim.FusedOptimizer) on the GPU: arithmetic against torch.optim (fp64
arbiter), torch-format checkpoints both ways, schedulers under graph replay, the graphed training iteration against the
eager one, the skip guard, eval after graphed training, training, and two ranks."""
import copy
import os
import socket
import sys

import pytest
import torch

import optim_cases as oc

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))


def _ours(kind, wd, params, odd_views=True):
    """FusedOptimizer over CUDA copies of `params`; the gradients are views into one flat buffer, every other one at an
    odd element offset (scalar path), the rest 16-byte aligned (vector path)."""
    from lanedetection_end2end_b200.optim import FusedOptimizer
    ps = [p.cuda().clone() for p in params]
    offs, off = [], 0
    for i, p in enumerate(ps):
        off += (1 if (odd_views and i % 2) else 0)
        offs.append(off)
        off = (off + p.numel() + 3) // 4 * 4
    flat = torch.zeros(off + 4, device="cuda")
    views = [flat[o:o + p.numel()].view_as(p) for o, p in zip(offs, ps)]
    return ps, views, FusedOptimizer(ps, kind, oc.LR[kind], wd)


def _feed(ps, views, gs):
    for p, v, g in zip(ps, views, gs):
        if g is None:
            p.grad = None
        else:
            v.copy_(g)
            p.grad = v


def _run_ours(opt, ps, views, grads):
    for gs in grads:
        _feed(ps, views, gs)
        opt.step()


def _check_gate(ours, t32, t64):
    assert set(ours) == set(t64)
    for name, x64 in t64.items():
        e_ours, e_t32 = oc.rel_err(ours[name], x64), oc.rel_err(t32[name], x64)
        assert e_ours <= 2 * e_t32 + 1e-7, (name, e_ours, e_t32)


@pytest.mark.parametrize("wd", [0.0, 1e-4])
@pytest.mark.parametrize("kind", ["adam", "sgd", "rmsprop"])
def test_arithmetic_against_torch_optim(kind, wd):
    params, grads = oc.make_params(), oc.make_grads()
    ps, views, opt = _ours(kind, wd, params)
    _run_ours(opt, ps, views, grads)
    p32, o32 = oc.torch_run(kind, wd, params, grads, torch.float32, "cuda", oc.STEPS)
    p64, o64 = oc.torch_run(kind, wd, params, grads, torch.float64, "cuda", oc.STEPS)
    ours = oc.tensors_of(ps, opt, kind)
    _check_gate(ours, oc.tensors_of(p32, o32, kind), oc.tensors_of(p64, o64, kind))
    assert torch.equal(ps[oc.NONE_GRAD].cpu(), params[oc.NONE_GRAD]) and not opt.state[ps[oc.NONE_GRAD]]
    assert opt.step_count == oc.STEPS and opt.skipped == 0
    # one step: every element within 2 ulp of torch's fp32 (foreach) result; report the bit-identical share
    ps1, views1, opt1 = _ours(kind, wd, params)
    _run_ours(opt1, ps1, views1, grads[:1])
    q32, r32 = oc.torch_run(kind, wd, params, grads, torch.float32, "cuda", 1)
    same = total = 0
    one = oc.tensors_of(ps1, opt1, kind)
    for name, x in oc.tensors_of(q32, r32, kind).items():
        assert oc.ulp_distance(one[name], x) <= 2, name
        same += int((one[name].view(torch.int32) == x.view(torch.int32)).sum())
        total += x.numel()
    share30 = sum(int((ours[n].view(torch.int32) == x.view(torch.int32)).sum())
                  for n, x in oc.tensors_of(p32, o32, kind).items()) / sum(x.numel() for x in ours.values())
    print("\nbit-identical to torch foreach fp32: %s wd=%g  1 step %.4f  30 steps %.4f" % (kind, wd, same / total, share30))


@pytest.mark.parametrize("kind", ["adam", "sgd", "rmsprop"])
def test_checkpoints_move_both_ways(kind):
    cls, extra = oc.KINDS[kind]
    wd = 1e-4
    params, grads = oc.make_params(), oc.make_grads(steps=15)
    p32, o32 = oc.torch_run(kind, wd, params, grads, torch.float32, "cuda", 15)
    p64, o64 = oc.torch_run(kind, wd, params, grads, torch.float64, "cuda", 15)
    t32, t64 = oc.tensors_of(p32, o32, kind), oc.tensors_of(p64, o64, kind)
    # ours for 5 steps -> torch for 10
    ps, views, opt = _ours(kind, wd, params)
    _run_ours(opt, ps, views, grads[:5])
    sd = opt.state_dict()
    tq = [p.clone() for p in ps]
    tor = cls(tq, lr=oc.LR[kind], weight_decay=wd, **extra)
    ref_sd = copy.deepcopy(o32.state_dict())
    tor.load_state_dict(sd)
    assert list(sd["param_groups"][0]) == list(ref_sd["param_groups"][0])
    assert set(sd["state"]) == set(ref_sd["state"])
    for i, st in sd["state"].items():
        assert list(st) == list(ref_sd["state"][i])
        if "step" in st:
            assert st["step"].device.type == "cpu" and st["step"].dtype == torch.float32 and float(st["step"]) == 5.0
    for gs in grads[5:]:
        for p, g in zip(tq, gs):
            p.grad = None if g is None else g.cuda()
        tor.step()
    _check_gate(oc.tensors_of(tq, tor, kind), t32, t64)
    # torch for 5 steps -> ours for 10
    q5, o5 = oc.torch_run(kind, wd, params, grads, torch.float32, "cuda", 5)
    ps2, views2, opt2 = _ours(kind, wd, [q.cpu() for q in q5])
    opt2.load_state_dict(o5.state_dict())
    _run_ours(opt2, ps2, views2, grads[5:])
    _check_gate(oc.tensors_of(ps2, opt2, kind), t32, t64)
    assert opt2.step_count == 15 or kind == "sgd"


def test_schedulers_reach_the_replayed_graph():
    from torch.optim import lr_scheduler
    params, grads = oc.make_params(), oc.make_grads(steps=12)
    ps, views, opt = _ours("sgd", 0.0, params, odd_views=False)
    tq = [p.cuda().clone() for p in params]
    tor = torch.optim.SGD(tq, lr=oc.LR["sgd"], momentum=0.9)
    _feed(ps, views, grads[0])
    opt.prepare(opt.grad_params())
    opt.sync_hyperparameters()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        opt.launch()
    scheds = [(lr_scheduler.StepLR(opt, 2, 0.5), lr_scheduler.StepLR(tor, 2, 0.5)),
              (lr_scheduler.LambdaLR(opt, lambda e: 1.0 / (1 + e)), lr_scheduler.LambdaLR(tor, lambda e: 1.0 / (1 + e))),
              (lr_scheduler.ReduceLROnPlateau(opt, factor=0.1, patience=0), lr_scheduler.ReduceLROnPlateau(tor, factor=0.1, patience=0))]
    lrs = []
    for it, gs in enumerate(grads):
        _feed(ps, views, gs)
        for p, gg in zip(tq, gs):
            p.grad = None if gg is None else gg.cuda()
        opt.sync_hyperparameters()
        g.replay()
        tor.step()
        a, b = scheds[it // 4]
        if isinstance(a, lr_scheduler.ReduceLROnPlateau):
            a.step(1.0)
            b.step(1.0)
        else:
            a.step()
            b.step()
        lrs.append(opt.param_groups[0]["lr"])
    torch.cuda.synchronize()
    assert len(set(lrs)) > 4
    for p, q in zip(ps, tq):
        assert torch.allclose(p, q, rtol=1e-6, atol=1e-9)


# ---------------------------------------------------------------------------------------------------------------------
# the model
# ---------------------------------------------------------------------------------------------------------------------
def _model(seed=21, L=2, B=2):
    from oracle import golden_check, inputs
    from lanedetection_end2end_b200.Loss_crit import backprojection_loss
    model, args = golden_check.build_net(L, 2, 0.3, B)
    sd = model.state_dict()
    for k, v in inputs.make_erfnet_params(3, L, seed=seed).items():
        sd[k] = torch.from_numpy(v)
    model.load_state_dict(sd)
    model = model.cuda().train()
    for m in model.modules():
        if hasattr(m, "dropout"):
            m.dropout.p = 0
    return model, backprojection_loss(args), L, B


def _batch(B, seed=40):
    from oracle import inputs
    x = torch.from_numpy(inputs.make_images(B, 256, 512, seed=seed)).cuda()
    xgt_np, valid_np = inputs.make_loss_targets(B, 4, seed=seed + 10)
    return x, torch.from_numpy(xgt_np).cuda(), torch.from_numpy(valid_np).cuda()


def _state_tensors(model, opt):
    out = {n: p.detach().clone() for n, p in model.named_parameters()}
    for n, p in model.named_parameters():
        for k, v in opt.state.get(p, {}).items():
            if k != "step":
                out[n + "." + k] = v.clone()
    return out


def test_graphed_iteration_equals_eager_iterations():
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.Loss_crit import fused_backprojection_loss
    from lanedetection_end2end_b200.optim import FusedOptimizer
    model, crit, L, B = _model()
    model2 = copy.deepcopy(model)
    x, xgt, valid = _batch(B)
    opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 1e-4)
    for _ in range(5):
        opt.zero_grad()
        out = model(x, torch.zeros(B, 4), True)
        loss, _ = fused_backprojection_loss(crit, out[:L], xgt, valid)
        loss.backward()
        opt.step()
    opt2 = FusedOptimizer(model2.parameters(), "adam", 1e-3, 1e-4)
    step = GraphedTrainStep(model2, crit, L, x, xgt, valid, optimizer=opt2)
    for _ in range(5):
        step()
    torch.cuda.synchronize()
    a, b = _state_tensors(model, opt), _state_tensors(model2, opt2)
    assert set(a) == set(b) and len(a) > len(list(model.parameters()))
    for n in a:
        assert torch.equal(a[n], b[n]), n
    assert opt.step_count == opt2.step_count == 5


def test_checkpoint_loaded_after_capture_reaches_the_replays():
    """Loading copies into the state tensors the captured segment table points at: replays after a load continue the
    loaded run exactly as the eager run does."""
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.Loss_crit import fused_backprojection_loss
    from lanedetection_end2end_b200.optim import FusedOptimizer
    model, crit, L, B = _model()
    model2 = copy.deepcopy(model)
    x, xgt, valid = _batch(B)
    opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 1e-4)

    def eager(n):
        for _ in range(n):
            opt.zero_grad()
            out = model(x, torch.zeros(B, 4), True)
            fused_backprojection_loss(crit, out[:L], xgt, valid)[0].backward()
            opt.step()
    eager(3)
    model_sd, opt_sd = copy.deepcopy(model.state_dict()), copy.deepcopy(opt.state_dict())
    opt2 = FusedOptimizer(model2.parameters(), "adam", 1e-3, 1e-4)
    step = GraphedTrainStep(model2, crit, L, x, xgt, valid, optimizer=opt2)
    for _ in range(2):                     # a different run, then the checkpoint of the eager one
        step()
    state_ptrs = [t.data_ptr() for st in opt2.state.values() for k, t in st.items() if k != "step"]
    model2.load_state_dict(model_sd)
    opt2.load_state_dict(opt_sd)
    assert [t.data_ptr() for st in opt2.state.values() for k, t in st.items() if k != "step"] == state_ptrs
    for _ in range(2):
        step()
    eager(2)
    torch.cuda.synchronize()
    a, b = _state_tensors(model, opt), _state_tensors(model2, opt2)
    for n in a:
        assert torch.equal(a[n], b[n]), n
    assert opt.step_count == opt2.step_count == 5


def test_skip_guard_operator_level():
    params, grads = oc.make_params(), oc.make_grads(steps=3)
    ps, views, opt = _ours("adam", 1e-4, params)
    _run_ours(opt, ps, views, grads[:2])
    _feed(ps, views, grads[2])
    status = torch.ones(1, dtype=torch.int32, device="cuda")
    before = {k: v.clone() for k, v in oc.tensors_of(ps, opt, "adam").items()}
    opt.launch(status=status)
    after = oc.tensors_of(ps, opt, "adam")
    assert all(torch.equal(before[k].view(torch.int32), after[k].view(torch.int32)) for k in before)
    assert opt.step_count == 2 and opt.skipped == 1
    status.zero_()
    opt.launch(status=status)
    assert opt.step_count == 3 and opt.skipped == 1
    assert not torch.equal(before["p0"], ps[0])


def test_skip_guard_in_the_graphed_iteration():
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.optim import FusedOptimizer
    model, crit, L, B = _model()
    x, xgt, valid = _batch(B)
    opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 0)
    step = GraphedTrainStep(model, crit, L, x, xgt, valid, optimizer=opt)
    step()
    torch.cuda.synchronize()
    assert opt.step_count == 1 and opt.skipped == 0
    oc_ = model.net.decoder.output_conv
    saved = (oc_.weight.detach().clone(), oc_.bias.detach().clone())
    with torch.no_grad():
        oc_.weight.zero_()
        oc_.bias.zero_()
    before = _state_tensors(model, opt)
    step()
    torch.cuda.synchronize()
    assert int(model.lsq_status.item()) != 0
    assert opt.step_count == 1 and opt.skipped == 1
    after = _state_tensors(model, opt)
    for n in before:
        assert torch.equal(before[n], after[n]), n
    with torch.no_grad():
        oc_.weight.copy_(saved[0])
        oc_.bias.copy_(saved[1])
    step()
    torch.cuda.synchronize()
    assert int(model.lsq_status.item()) == 0
    assert opt.step_count == 2 and opt.skipped == 1
    assert not torch.equal(before["net.decoder.output_conv.weight"], oc_.weight)


def test_eval_after_graphed_training_sees_the_trained_weights():
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.optim import FusedOptimizer
    model, crit, L, B = _model()
    x, xgt, valid = _batch(B)
    with torch.no_grad():                       # builds and caches the BatchNorm-folded eval operands
        model.eval()(x, torch.zeros(B, 4), True)
    model.train()
    opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 0)
    step = GraphedTrainStep(model, crit, L, x, xgt, valid, optimizer=opt)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    fresh, _, _, _ = _model(seed=99)
    fresh.load_state_dict(model.state_dict())
    with torch.no_grad():
        got = model.eval()(x, torch.zeros(B, 4), True)
        want = fresh.eval()(x, torch.zeros(B, 4), True)
    for i in list(range(L)) + [5]:
        assert torch.equal(got[i], want[i]), i


def test_training_with_the_fused_optimizer():
    import train_synthetic
    for graphed in (False, True):
        rep = train_synthetic.run(steps=40, batch=4, fused=True, graphed=graphed)
        assert rep["skipped"] == 0, (graphed, rep)
        assert rep["loss_last"] < 0.5 * rep["loss_first"], (graphed, rep)
        assert all(v == v and v < 1e12 for v in rep["losses"]), (graphed, rep)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from lanedetection_end2end_b200.ddp import FlatGradAllReduce, broadcast_parameters
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.optim import FusedOptimizer
    model, crit, L, B = _model()
    broadcast_parameters(model)
    opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 1e-4)
    step = GraphedTrainStep(model, crit, L, *_batch(B, seed=40 + rank), FlatGradAllReduce(model),
                            capture_error_mode="thread_local", optimizer=opt)
    step()
    step()
    # a singular system on rank 1 only: every rank must skip, or the replicas would part
    oc_ = model.net.decoder.output_conv
    saved = (oc_.weight.detach().clone(), oc_.bias.detach().clone())
    if rank == 1:
        with torch.no_grad():
            oc_.weight.zero_()
            oc_.bias.zero_()
    step()
    torch.cuda.synchronize()
    local = int(model.lsq_status.item())
    with torch.no_grad():
        oc_.weight.copy_(saved[0])
        oc_.bias.copy_(saved[1])
    step()
    torch.cuda.synchronize()
    q.put((rank, torch.cat([p.detach().reshape(-1) for p in model.parameters()]).cpu(), opt.step_count, opt.skipped, local))
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_stay_bit_identical():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_rank_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict((r[0], r[1:]) for r in (q.get(timeout=600) for _ in range(2)))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert res[0][3] == 0 and res[1][3] != 0           # only rank 1 saw the singular system ...
    assert res[0][1:3] == res[1][1:3] == (3, 1)         # ... and both ranks skipped that update
    assert torch.equal(res[0][0].view(torch.int32), res[1][0].view(torch.int32))
