"""Shared inputs and error measure of the optimizer tests (test_optim_cpu.py, test_optim_gpu.py): parameter tensors with
shapes of the model, 30 recorded gradient steps whose per-tensor scales run from 1e-6 to 1e2, and torch.optim runs on
float64 copies as the arbiter."""
import torch

# shapes of the model's parameters (ERFNet convolutions, biases, BatchNorm affines, output_conv)
SHAPES = [(16, 3, 3, 3), (16,), (48, 16, 3, 3), (64,), (64, 64, 3, 1), (64,), (64, 64, 1, 3), (128, 128, 3, 1), (128,),
          (128, 128, 1, 3), (128, 64, 3, 3), (16,), (64, 16, 3, 3), (16, 2, 2, 2), (2,), (5,)]
NONE_GRAD = len(SHAPES) - 1          # this parameter never gets a gradient (like net.encoder.output_conv)
STEPS = 30
KINDS = {"adam": (torch.optim.Adam, {}), "sgd": (torch.optim.SGD, {"momentum": 0.9}),
         "rmsprop": (torch.optim.RMSprop, {"momentum": 0.9})}
LR = {"adam": 1e-3, "sgd": 1e-2, "rmsprop": 1e-3}
STATE_NAMES = {"adam": ("exp_avg", "exp_avg_sq"), "sgd": ("momentum_buffer",), "rmsprop": ("square_avg", "momentum_buffer")}


def make_params(seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g, dtype=torch.float32) * 0.1 for s in SHAPES]


def make_grads(seed=1, steps=STEPS):
    """grads[step][tensor] (fp32, None for NONE_GRAD); tensor i has scale 10^(-6 + 8 i / (n - 2))."""
    g = torch.Generator().manual_seed(seed)
    n = len(SHAPES)
    scales = [10.0 ** (-6 + 8 * i / (n - 2)) for i in range(n)]
    return [[None if i == NONE_GRAD else torch.randn(s, generator=g, dtype=torch.float32) * scales[i]
             for i, s in enumerate(SHAPES)] for _ in range(steps)]


def rel_err(x, x64):
    d = float((x.double().cpu() - x64.cpu()).abs().max())
    m = float(x64.abs().max())
    return d / m if m > 0 else d


def torch_run(kind, wd, params, grads, dtype, device, steps, state_dict=None, **kw):
    """torch.optim.<Cls> over copies of `params` in `dtype` on `device`, fed `grads[:steps]`; returns (params, optimizer)."""
    cls, extra = KINDS[kind]
    ps = [p.detach().to(device=device, dtype=dtype).clone() for p in params]
    opt = cls(ps, lr=LR[kind], weight_decay=wd, **extra, **kw)
    if state_dict is not None:
        opt.load_state_dict(state_dict)
    for gs in grads[:steps]:
        for p, g in zip(ps, gs):
            p.grad = None if g is None else g.to(device=device, dtype=dtype)
        opt.step()
    return ps, opt


def tensors_of(ps, opt, kind):
    """{name: tensor} of every parameter and state tensor (parameters without state contribute the parameter only)."""
    out = {}
    for i, p in enumerate(ps):
        out["p%d" % i] = p
        st = opt.state.get(p, {})
        for k in STATE_NAMES[kind]:
            if k in st:
                out["p%d.%s" % (i, k)] = st[k]
    return out


def ulp_distance(a, b):
    """max distance in units in the last place between two fp32 tensors (ordered-integer view of the bits)."""
    def ordered(x):
        i = x.contiguous().float().cpu().view(torch.int32).long()
        return torch.where(i < 0, -(i & 0x7fffffff), i)
    return int((ordered(a) - ordered(b)).abs().max())
