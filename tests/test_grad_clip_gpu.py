"""Gradient clipping in the fused optimizer on the GPU (csrc/optim.cu: lf_grad_norm, lf_optim_step_clip,
lf_optim_step_pp_clip; optim.FusedOptimizer(max_grad_norm=...)): the norm against fp64, its repeatability and its
independence of the load path, the coefficient against torch's clip_grads_with_norm_ on the device, the clipped update bit
for bit against the unclipped one fed torch-scaled gradients and against torch.optim at the fp32 / fp64 gates, the skip of
non-finite gradients, the graphed step, the training epochs, and two ranks."""
import copy
import math
import os
import sys

import pytest
import torch

import optim_cases as oc
from test_epoch_gpu import (criteria, eager_train, loaders, make_args, make_model, paths, per_lane_loss,  # noqa: F401
                            Listed)
from test_optim_gpu import _batch, _check_gate, _free_port, _model, _state_tensors

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
KINDS = ["adam", "sgd", "rmsprop"]


def _ours(kind, wd, params, pp=False, max_norm=None, odd_views=True):
    """FusedOptimizer over CUDA copies of `params`; the gradients are views into one flat buffer, every other one at an
    odd element offset (scalar path), the rest 16-byte aligned (vector path), as test_optim_gpu._ours builds them."""
    from lanedetection_end2end_b200.optim import FusedOptimizer
    ps = [p.cuda().clone() for p in params]
    offs, off = [], 0
    for i, p in enumerate(ps):
        off += (1 if (odd_views and i % 2) else 0)
        offs.append(off)
        off = (off + p.numel() + 3) // 4 * 4
    flat = torch.zeros(off + 4, device="cuda")
    views = [flat[o:o + p.numel()].view_as(p) for o, p in zip(offs, ps)]
    return ps, views, FusedOptimizer(ps, kind, oc.LR[kind], wd, per_param_step=pp, max_grad_norm=max_norm)


def _feed(ps, views, gs):
    for p, v, g in zip(ps, views, gs):
        if g is None:
            p.grad = None
        else:
            v.copy_(g)
            p.grad = v


def _norm_only(opt):
    """The norm launch alone over the optimizer's prepared table; returns (total_norm, clip_coef, nonfinite) bits."""
    from lanedetection_end2end_b200 import _capi
    opt.prepare(opt.grad_params())
    opt.sync_hyperparameters()
    _capi.call("lf_grad_norm_pp" if opt.per_param_step else "lf_grad_norm", _capi.ptr(opt._table), opt._nsegs,
               opt._nchunks, _capi.ptr(opt._clip), _capi.ptr(opt._norm_ws), opt._norm_ws.numel() * 8,
               _capi.stream_ptr())
    w = opt._clip.view(torch.int32)[:4].cpu()
    return int(w[1]), int(w[2]), int(w[3])


def _f32(bits):
    return torch.tensor([bits], dtype=torch.int32).view(torch.float32).item()


def _norm64(grads):
    return torch.linalg.vector_norm(torch.cat([g.double().reshape(-1).cuda() for g in grads if g is not None]))


def _check_norm(grads, shapes, max_norm=1.0):
    """lf_grad_norm over `grads` (odd-offset and aligned views, both step modes): within 1 fp32 ulp of the fp64 norm,
    bit-identical over repeated launches, and the same bits whichever load path each tensor takes."""
    n64 = _norm64(grads)
    seen = set()
    for odd in (True, False):
        for pp in (False, True):
            ps, views, opt = _ours("adam", 0.0, [torch.zeros(s) for s in shapes], pp=pp, max_norm=max_norm,
                                   odd_views=odd)
            _feed(ps, views, grads)
            for _ in range(3):
                seen.add(_norm_only(opt))
    assert len(seen) == 1, seen
    norm_bits, _, nonfinite = seen.pop()
    got = torch.tensor([_f32(norm_bits)], dtype=torch.float32)
    assert nonfinite == 0
    assert oc.ulp_distance(got, n64.float().reshape(1)) <= 1, (float(got), float(n64))
    return float(got)


def test_norm_of_the_optim_cases():
    for step in oc.make_grads(steps=3):
        _check_norm(step, oc.SHAPES)


def test_norm_of_clas_shaped_parameters():
    """The --clas model's parameter shapes (7.3 M elements), per-tensor scales from 1e-6 to 1e2."""
    import bench
    import bench_train_iter
    model, _ = bench_train_iter._model(dict(bench.CONFIGS[2], clas=True))
    shapes = [p.shape for n, p in model.named_parameters() if "encoder.output_conv" not in n]
    del model
    g = torch.Generator(device="cuda").manual_seed(3)
    grads = [torch.randn(s, device="cuda", generator=g) * 10.0 ** (-6 + 8 * (i % 9) / 8) for i, s in enumerate(shapes)]
    assert sum(x.numel() for x in grads) > 7_000_000
    _check_norm(grads, shapes)


@pytest.mark.parametrize("case", ["active", "inactive", "zero", "zero_active"])
def test_coefficient_equals_torch_clip_on_the_device(case):
    grads = oc.make_grads(steps=1)[0]
    if case.startswith("zero"):
        grads = [None if g is None else torch.zeros_like(g) for g in grads]
    n64 = float(_norm64(grads))
    max_norm = {"active": 0.37 * n64, "inactive": 2.5 * n64, "zero": 1.0, "zero_active": 1e-9}[case]
    ps, views, opt = _ours("sgd", 0.0, oc.make_params(), max_norm=max_norm)
    _feed(ps, views, grads)
    _, coef_bits, _ = _norm_only(opt)
    p = torch.zeros(3, device="cuda", requires_grad=True)
    p.grad = torch.ones(3, device="cuda")
    torch.nn.utils.clip_grads_with_norm_([p], max_norm, opt.grad_norm.clone())
    want = p.grad.view(torch.int32)
    assert bool((want == coef_bits).all()), (case, _f32(coef_bits), p.grad)
    coef = _f32(coef_bits)
    assert (coef < 1) == (case in ("active", "zero_active")), coef


def _torch_clipped_run(kind, wd, params, grads, dtype, max_norm):
    cls, extra = oc.KINDS[kind]
    ps = [p.detach().to(device="cuda", dtype=dtype).clone() for p in params]
    opt = cls(ps, lr=oc.LR[kind], weight_decay=wd, **extra)
    for gs in grads:
        for p, g in zip(ps, gs):
            p.grad = None if g is None else g.to(device="cuda", dtype=dtype)
        torch.nn.utils.clip_grad_norm_([p for p in ps if p.grad is not None], max_norm)
        opt.step()
    return oc.tensors_of(ps, opt, kind)


def _counts(opt):
    return opt.step_counts, opt.skipped, opt.nonfinite_skipped


@pytest.mark.parametrize("pp", [False, True])
@pytest.mark.parametrize("wd", [0.0, 1e-4])
@pytest.mark.parametrize("kind", KINDS)
def test_clipped_update(kind, wd, pp):
    steps = 8
    params, grads = oc.make_params(), oc.make_grads(steps=steps)
    norms = sorted(float(_norm64(gs)) for gs in grads)
    max_norm = 0.5 * (norms[steps // 2 - 1] + norms[steps // 2])         # clips about half of the steps
    # ours, clipping
    ps, views, opt = _ours(kind, wd, params, pp=pp, max_norm=max_norm)
    # the unclipped optimizer fed the gradients that torch's clip_grads_with_norm_ scaled by our norm
    qs, qviews, ref = _ours(kind, wd, params, pp=pp)
    clipped = 0
    for gs in grads:
        _feed(ps, views, gs)
        opt.step()
        norm = opt.grad_norm.clone()
        clipped += int(float(norm) > max_norm)
        _feed(qs, qviews, gs)
        torch.nn.utils.clip_grads_with_norm_([q for q in qs if q.grad is not None], max_norm, norm)
        ref.step()
        for v, g in zip(views, gs):                # p.grad is not rewritten
            assert g is None or torch.equal(v.cpu(), g)
    assert 0 < clipped < steps
    a, b = oc.tensors_of(ps, opt, kind), oc.tensors_of(qs, ref, kind)
    assert set(a) == set(b)
    for n in a:
        assert torch.equal(a[n].view(torch.int32), b[n].view(torch.int32)), n
    assert _counts(opt) == _counts(ref) and opt.skipped == 0 and opt.nonfinite_skipped == 0
    # torch.optim after clip_grad_norm_, fp32 and fp64
    t32 = _torch_clipped_run(kind, wd, params, grads, torch.float32, max_norm)
    t64 = _torch_clipped_run(kind, wd, params, grads, torch.float64, max_norm)
    _check_gate(a, t32, t64)
    # a threshold above every norm: exactly the unclipped bits
    ps2, views2, big = _ours(kind, wd, params, pp=pp, max_norm=1e30)
    qs2, qviews2, plain = _ours(kind, wd, params, pp=pp)
    for gs in grads:
        _feed(ps2, views2, gs)
        big.step()
        _feed(qs2, qviews2, gs)
        plain.step()
    a, b = oc.tensors_of(ps2, big, kind), oc.tensors_of(qs2, plain, kind)
    for n in a:
        assert torch.equal(a[n].view(torch.int32), b[n].view(torch.int32)), n


@pytest.mark.parametrize("pp", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_nonfinite_gradient_skips_the_update(kind, pp):
    params, grads = oc.make_params(), oc.make_grads(steps=5)
    k = 2
    bad = [None if g is None else g.clone() for g in grads[k]]
    bad[3].view(-1)[7] = float("inf")
    bad[10].view(-1)[5] = float("nan")
    max_norm = 0.5 * float(_norm64(grads[0]))
    ps, views, opt = _ours(kind, 1e-4, params, pp=pp, max_norm=max_norm)
    qs, qviews, ref = _ours(kind, 1e-4, params, pp=pp, max_norm=max_norm)       # never sees step k
    for t, gs in enumerate(grads):
        if t == k:
            _feed(ps, views, bad)
            before = {n: x.clone() for n, x in oc.tensors_of(ps, opt, kind).items()}
            counts = _counts(opt)
            opt.step()
            after = oc.tensors_of(ps, opt, kind)
            assert set(before) == set(after)
            for n in before:
                assert torch.equal(before[n].view(torch.int32), after[n].view(torch.int32)), n
            steps, skipped, nonfinite = _counts(opt)
            assert steps == counts[0] and skipped == counts[1] + 1 and nonfinite == counts[2] + 1
            assert not math.isfinite(float(opt.grad_norm))
            continue
        _feed(ps, views, gs)
        opt.step()
        _feed(qs, qviews, gs)
        ref.step()
    a, b = oc.tensors_of(ps, opt, kind), oc.tensors_of(qs, ref, kind)
    for n in a:
        assert torch.equal(a[n].view(torch.int32), b[n].view(torch.int32)), n
    assert opt.step_counts == ref.step_counts and opt.skipped == opt.nonfinite_skipped == 1 and ref.skipped == 0


# ---------------------------------------------------------------------------------------------------------------------
# the graphed step
# ---------------------------------------------------------------------------------------------------------------------
def test_graphed_iteration_equals_eager_iterations_with_clipping():
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.Loss_crit import fused_backprojection_loss
    from lanedetection_end2end_b200.optim import FusedOptimizer
    model, crit, L, B = _model()
    model2 = copy.deepcopy(model)
    x, xgt, valid = _batch(B)
    m1, m2 = 1e-4, 1e12                # clipping, then a threshold above every norm (they are about 1e6)
    opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 1e-4, max_grad_norm=m1)
    opt2 = FusedOptimizer(model2.parameters(), "adam", 1e-3, 1e-4, max_grad_norm=m1)
    step = GraphedTrainStep(model2, crit, L, x, xgt, valid, optimizer=opt2)
    norms = []
    for it in range(6):
        if it == 3:
            opt.max_grad_norm = opt2.max_grad_norm = m2        # reaches the next replay without a recapture
        opt.zero_grad()
        out = model(x, torch.zeros(B, 4), True)
        fused_backprojection_loss(crit, out[:L], xgt, valid)[0].backward()
        opt.step()
        step()
        norms.append((float(opt.grad_norm), float(opt2.grad_norm)))
    torch.cuda.synchronize()
    assert all(a == b for a, b in norms) and all(m1 < n < m2 for n, _ in norms), norms
    a, b = _state_tensors(model, opt), _state_tensors(model2, opt2)
    assert set(a) == set(b) and len(a) > len(list(model.parameters()))
    for n in a:
        assert torch.equal(a[n], b[n]), n
    assert opt.step_count == opt2.step_count == 6
    # the graph holds the clipped launches: clipping cannot be turned off under it
    with pytest.raises(ValueError, match="cannot turn clipping off"):
        opt2.max_grad_norm = None
    assert opt2.max_grad_norm == m2


def test_singular_batch_is_skipped_by_the_status_word_not_as_nonfinite():
    from lanedetection_end2end_b200.engine import GraphedTrainStep
    from lanedetection_end2end_b200.optim import FusedOptimizer
    model, crit, L, B = _model()
    x, xgt, valid = _batch(B)
    opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 0, max_grad_norm=1e-3)
    step = GraphedTrainStep(model, crit, L, x, xgt, valid, optimizer=opt)
    step()
    torch.cuda.synchronize()
    assert opt.step_count == 1 and opt.skipped == 0 and opt.nonfinite_skipped == 0
    oc_ = model.net.decoder.output_conv
    saved = (oc_.weight.detach().clone(), oc_.bias.detach().clone())
    with torch.no_grad():
        oc_.weight.zero_()
        oc_.bias.zero_()
    before = _state_tensors(model, opt)
    step()
    torch.cuda.synchronize()
    assert int(model.lsq_status.item()) != 0
    assert opt.step_count == 1 and opt.skipped == 1 and opt.nonfinite_skipped == 0
    after = _state_tensors(model, opt)
    for n in before:
        assert torch.equal(before[n], after[n]), n
    with torch.no_grad():
        oc_.weight.copy_(saved[0])
        oc_.bias.copy_(saved[1])
    step()
    torch.cuda.synchronize()
    assert opt.step_count == 2 and opt.skipped == 1 and opt.nonfinite_skipped == 0


# ---------------------------------------------------------------------------------------------------------------------
# the training epochs
# ---------------------------------------------------------------------------------------------------------------------
class NonFinite:
    """Multiplies one parameter's gradient by NaN in the batches listed in `which` (a backward hook whose factor `wrap`
    sets on the stream before each batch is handed out, so eager and graphed runs see it)."""

    def __init__(self, param, which):
        self.which, self.scale = set(which), torch.ones((), device="cuda")
        self.h = param.register_hook(lambda g: g * self.scale)

    def wrap(self, batches):
        for k, b in enumerate(batches):
            self.scale.fill_(float("nan") if k in self.which else 1.0)
            yield b


def test_train_epoch_with_clipping_equals_eager_main(paths, capsys):
    from lanedetection_end2end_b200 import engine
    from lanedetection_end2end_b200.Networks import utils as nu
    args = make_args("clas4", paths[0])
    train, _, _ = loaders(paths, args)
    batches = list(train)
    batches = batches + batches[:1]
    crits = criteria(args)
    ma, mb = make_model(args), make_model(args)
    mb.load_state_dict(ma.state_dict())
    max_norm = 1e-3
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True, max_grad_norm=max_norm)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True, max_grad_norm=max_norm)
    hooks = [NonFinite(ma.net.decoder.output_conv.weight, [1]), NonFinite(mb.net.decoder.output_conv.weight, [1])]
    try:
        want_loss, want_rmse, _, _ = eager_train(Listed(batches, hooks[0].wrap), ma, oa, *crits, args, per_lane_loss)
        capsys.readouterr()
        got_loss, got_rmse = engine.train_epoch(Listed(batches, hooks[1].wrap), mb, ob, *crits, args, 0)
    finally:
        for h in hooks:
            h.h.remove()
    assert "1 of 3 updates skipped: non-finite gradients" in capsys.readouterr().out
    assert got_loss == want_loss and got_rmse == want_rmse
    assert float(ob.grad_norm) > max_norm and float(oa.grad_norm) == float(ob.grad_norm)
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k
    sa, sb = oa.state_dict(), ob.state_dict()
    assert sa["state"].keys() == sb["state"].keys()
    for k in sa["state"]:
        for name, t in sa["state"][k].items():
            assert torch.equal(t, sb["state"][k][name]), (k, name)
    assert oa.step_count == ob.step_count == 2 and oa.nonfinite_skipped == ob.nonfinite_skipped == 1
    # an epoch without a non-finite gradient prints no such line
    engine.train_epoch(batches[:2], mb, ob, *crits, args, 1)
    assert "non-finite" not in capsys.readouterr().out


def test_train_epoch_bev_with_clipping_equals_eager_main(tmp_path_factory):
    import test_epoch_bev_gpu as eb
    from lanedetection_end2end_b200 import engine
    from lanedetection_end2end_b200.Networks import utils as nu
    bev_paths = eb.paths.__wrapped__(tmp_path_factory)         # the BEV tests' fixture directory, built here
    args = eb.make_args("l2", bev_paths[0])
    batches = eb.batches_of(bev_paths, args, "train")
    crits = eb.criteria(args)
    ma, mb = eb.make_model(args), eb.make_model(args)
    mb.load_state_dict(ma.state_dict())
    oa = nu.define_optim("adam", ma.parameters(), 1e-3, 0, fused=True, max_grad_norm=1e-3)
    ob = nu.define_optim("adam", mb.parameters(), 1e-3, 0, fused=True, max_grad_norm=1e-3)
    want, _ = eb.eager_train(batches, ma, oa, crits[1], args)
    got = engine.train_epoch_bev(batches, mb, ob, *crits, args, 0)
    assert got == want, (got, want)
    assert float(ob.grad_norm) > 1e-3
    for (k, a), b in zip(ma.named_parameters(), mb.parameters()):
        assert torch.equal(a, b), k


# ---------------------------------------------------------------------------------------------------------------------
# two ranks
# ---------------------------------------------------------------------------------------------------------------------
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
    opt = FusedOptimizer(model.parameters(), "adam", 1e-3, 1e-4, max_grad_norm=1e-3)
    step = GraphedTrainStep(model, crit, L, *_batch(B, seed=40 + rank), FlatGradAllReduce(model),
                            capture_error_mode="thread_local", optimizer=opt)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    q.put((rank, torch.cat([p.detach().reshape(-1) for p in model.parameters()]).cpu(), opt.step_count,
           float(opt.grad_norm)))
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_stay_bit_identical_with_clipping():
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
    assert res[0][1:] == res[1][1:] and res[0][1] == 3 and res[0][2] > 1e-3
    assert torch.equal(res[0][0].view(torch.int32), res[1][0].view(torch.int32))
