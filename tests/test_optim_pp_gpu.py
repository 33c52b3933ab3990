"""FusedOptimizer(per_param_step=True) (csrc/optim.cu: lf_optim_step_pp) on the GPU: bit for bit against torch.optim's
foreach path in parameters, state and per-parameter step over a run whose set of parameters with a gradient changes
(a subset, more, fewer, the dropped ones back) and that includes a skipped update; the same run captured and replayed,
with the set changed between captures; torch-format checkpoints both ways with differing steps; the default mode next
to the new one on a fixed set, and its set-change refusal."""
import pytest
import torch

import optim_cases as oc
from test_optim_pp_cpu import _subset_grads

pytestmark = pytest.mark.gpu

STEPS = 12
SKIP_AT = 5           # the update of this step is skipped by a nonzero status word


def _ours(kind, wd, params, per_param_step=True):
    from lanedetection_end2end_b200.optim import FusedOptimizer
    ps = [p.cuda().clone() for p in params]
    grads = [torch.zeros_like(p) for p in ps]     # persistent gradient tensors (a captured table reads them by address)
    return ps, grads, FusedOptimizer(ps, kind, oc.LR[kind], wd, per_param_step=per_param_step)


def _feed(ps, gbufs, gs):
    for p, buf, g in zip(ps, gbufs, gs):
        if g is None:
            p.grad = None
        else:
            buf.copy_(g)
            p.grad = buf


def _torch_run(kind, wd, params, grads, skip=SKIP_AT):
    """torch.optim.<Cls>(foreach=True) on CUDA over `grads`, leaving out step `skip` (the reference skips that batch)."""
    cls, extra = oc.KINDS[kind]
    ps = [p.cuda().clone() for p in params]
    opt = cls(ps, lr=oc.LR[kind], weight_decay=wd, foreach=True, **extra)
    for t, gs in enumerate(grads):
        if t == skip:
            continue
        for p, g in zip(ps, gs):
            p.grad = None if g is None else g.cuda()
        opt.step()
    return ps, opt


def _want_steps(opt, ps, grads):
    """torch's per-parameter step (SGD: the number of updates, which torch does not keep)."""
    out = []
    for i, p in enumerate(ps):
        st = opt.state.get(p, {})
        if "step" in st:
            out.append(int(st["step"]))
        else:
            out.append(sum(1 for t, gs in enumerate(grads) if t != SKIP_AT and gs[i] is not None))
    return out


def _assert_bits(ours_ps, ours_opt, want_ps, want_opt, kind):
    a, b = oc.tensors_of(ours_ps, ours_opt, kind), oc.tensors_of(want_ps, want_opt, kind)
    assert set(a) == set(b)
    for n in b:
        assert torch.equal(a[n].view(torch.int32), b[n].view(torch.int32)), n


@pytest.mark.parametrize("wd", [0.0, 1e-4])
@pytest.mark.parametrize("kind", ["adam", "sgd", "rmsprop"])
def test_changing_parameter_set_equals_torch_bit_for_bit(kind, wd):
    params, grads = oc.make_params(), _subset_grads(STEPS)
    ps, gbufs, opt = _ours(kind, wd, params)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    for t, gs in enumerate(grads):
        _feed(ps, gbufs, gs)
        if t == SKIP_AT:
            before = {k: v.clone() for k, v in oc.tensors_of(ps, opt, kind).items()}
            counts = opt.step_counts
            status.fill_(1)
            opt.prepare(opt.grad_params())
            opt.sync_hyperparameters()
            opt.launch(status=status)
            status.zero_()
            after = oc.tensors_of(ps, opt, kind)
            assert all(torch.equal(before[k].view(torch.int32), after[k].view(torch.int32)) for k in before)
            assert opt.step_counts == counts and opt.skipped == 1
            continue
        opt.step()
    wp, wo = _torch_run(kind, wd, params, grads)
    _assert_bits(ps, opt, wp, wo, kind)
    want = _want_steps(wo, wp, grads)
    assert opt.step_counts == want and opt.step_count == max(want) and len(set(want)) > 2
    assert want[oc.NONE_GRAD] == 0 and not opt.state[ps[oc.NONE_GRAD]]
    if kind != "sgd":
        sd = opt.state_dict()
        assert {i: float(st["step"]) for i, st in sd["state"].items()} == \
            {i: float(st["step"]) for i, st in wo.state_dict()["state"].items()}


@pytest.mark.parametrize("kind", ["adam", "sgd", "rmsprop"])
def test_captured_replays_with_the_set_changed_between_captures(kind):
    """One graph per parameter set, captured when the set first appears and replayed whenever it comes back: the run
    equals torch's bit for bit, including the skipped update (a graph replayed with the status word set)."""
    wd = 1e-4
    params, grads = oc.make_params(), _subset_grads(STEPS)
    ps, gbufs, opt = _ours(kind, wd, params)
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    graphs = {}
    s = torch.cuda.Stream()
    for t, gs in enumerate(grads):
        _feed(ps, gbufs, gs)
        key = tuple(g is not None for g in gs)
        if key not in graphs:
            opt.prepare(opt.grad_params())
            opt.sync_hyperparameters()
            s.wait_stream(torch.cuda.current_stream())
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=s):
                opt.launch(status=status)
            torch.cuda.current_stream().wait_stream(s)
            graphs[key] = g
        status.fill_(1 if t == SKIP_AT else 0)
        graphs[key].replay()
    torch.cuda.synchronize()
    assert len(graphs) >= 3
    wp, wo = _torch_run(kind, wd, params, grads)
    _assert_bits(ps, opt, wp, wo, kind)
    assert opt.step_counts == _want_steps(wo, wp, grads) and opt.skipped == 1
    # a set change during capture is refused
    _feed(ps, gbufs, [g if i % 3 else None for i, g in enumerate(oc.make_grads(steps=1)[0])])
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="changed during CUDA graph capture"):
        with torch.cuda.graph(g, stream=s):
            opt.step()


@pytest.mark.parametrize("kind", ["adam", "sgd", "rmsprop"])
def test_checkpoints_with_differing_steps_move_both_ways(kind):
    cls, extra = oc.KINDS[kind]
    wd = 1e-4
    params, grads = oc.make_params(), _subset_grads(STEPS)
    grads = [gs for t, gs in enumerate(grads) if t != SKIP_AT]
    half = len(grads) // 2
    p_all, o_all = _torch_run(kind, wd, params, grads, skip=None)
    # ours for the first half -> torch for the rest
    ps, gbufs, opt = _ours(kind, wd, params)
    for gs in grads[:half]:
        _feed(ps, gbufs, gs)
        opt.step()
    sd = opt.state_dict()
    tq = [p.clone() for p in ps]
    tor = cls(tq, lr=oc.LR[kind], weight_decay=wd, foreach=True, **extra)
    tor.load_state_dict(sd)
    for gs in grads[half:]:
        for p, g in zip(tq, gs):
            p.grad = None if g is None else g.cuda()
        tor.step()
    _assert_bits(tq, tor, p_all, o_all, kind)
    # torch for the first half -> ours for the rest
    q, oq = _torch_run(kind, wd, params, grads[:half], skip=None)
    ps2, gbufs2, opt2 = _ours(kind, wd, [x.cpu() for x in q])
    opt2.load_state_dict(oq.state_dict())
    for gs in grads[half:]:
        _feed(ps2, gbufs2, gs)
        opt2.step()
    _assert_bits(ps2, opt2, p_all, o_all, kind)
    if kind != "sgd":
        assert opt2.step_counts == [int(o_all.state[p]["step"]) if p in o_all.state else 0 for p in p_all]


def test_default_mode_unchanged_next_to_per_parameter_mode():
    """On a fixed set both modes give torch's bits; the default mode still refuses a changing set."""
    params, grads = oc.make_params(), oc.make_grads(steps=10)
    runs = {}
    for pp in (False, True):
        ps, gbufs, opt = _ours("adam", 1e-4, params, per_param_step=pp)
        for gs in grads:
            _feed(ps, gbufs, gs)
            opt.step()
        runs[pp] = (ps, opt)
    (pa, oa), (pb, ob) = runs[False], runs[True]
    for n, x in oc.tensors_of(pa, oa, "adam").items():
        assert torch.equal(x.view(torch.int32), oc.tensors_of(pb, ob, "adam")[n].view(torch.int32)), n
    assert oa.step_count == ob.step_count == 10
    assert oa.step_counts == ob.step_counts == [0 if i == oc.NONE_GRAD else 10 for i in range(len(pa))]
    wp, wo = _torch_run("adam", 1e-4, params, grads, skip=None)
    _assert_bits(pa, oa, wp, wo, "adam")
    gs = list(grads[0])
    gs[0] = None
    _feed(pa, [torch.zeros_like(p) for p in pa], gs)
    with pytest.raises(ValueError, match="keeps one step count for all parameters"):
        oa.step()
