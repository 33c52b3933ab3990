"""Optimizer update on the library's kernel (csrc/optim.cu: lf_optim_step): the Adam / SGD / RMSprop that the reference's
``define_optim`` builds (BP/Networks/utils.py:451-461, stepped at BP/main.py:262,340), as ONE launch over every parameter
that has a gradient.

The step counter, the hyperparameters and a count of skipped updates live in device memory, so the update can be captured
into the training step's CUDA graph (engine.GraphedTrainStep(..., optimizer=...)): a scheduler's new ``lr`` reaches the next
replay without a recapture, and a guarded launch reads the LSQ status word on the device and leaves everything unchanged
for a batch with a singular system, as the reference's skip of that batch does (BP/main.py:289-292).

``state_dict()`` / ``load_state_dict()`` use torch.optim's format exactly (``param_groups`` key for key, per-parameter
``step`` as a CPU float32 tensor, independent state tensors), so checkpoints move both ways between this class and
``torch.optim.<Cls>``.  By default all parameters share one step count (csrc/optim.cu: lf_optim_step), so the set of
parameters with a gradient must not change.  ``per_param_step=True`` keeps one device count per parameter
(lf_optim_step_pp), as torch.optim does: the set may change between updates, which a --pretrained run does by
construction (its segmentation epochs train ``output_conv2``, its end-to-end epochs ``output_conv`` and the heads).
"""
import ctypes

import torch

from . import _capi

ptr = _capi.ptr

# kind -> (torch class whose semantics and state format are kept, constructor arguments of define_optim, kernel id)
_KINDS = {
    "adam": (torch.optim.Adam, {}, _capi.OPTIM_ADAM),
    "sgd": (torch.optim.SGD, {"momentum": 0.9}, _capi.OPTIM_SGD),
    "rmsprop": (torch.optim.RMSprop, {"momentum": 0.9}, _capi.OPTIM_RMSPROP),
}
# per-parameter state tensors in torch's order: LfOptimSeg.state0, .state1
STATE_KEYS = {"adam": ("exp_avg", "exp_avg_sq"), "sgd": ("momentum_buffer",), "rmsprop": ("square_avg", "momentum_buffer")}
_UNSUPPORTED = ("amsgrad", "nesterov", "centered", "maximize")


class FusedOptimizer(torch.optim.Optimizer):
    """``FusedOptimizer(params, kind, lr, weight_decay, per_param_step=False)`` with kind in {"adam", "sgd", "rmsprop"}:
    the arguments and semantics of ``define_optim(kind, params, lr, weight_decay)`` (SGD and RMSprop with momentum 0.9),
    one parameter group.

    ``step()`` updates the parameters whose ``.grad`` is not None, in one launch on the current stream, without a host
    synchronisation.  ``skipped`` / ``step_count`` / ``step_counts`` read the device counters (one synchronisation each).

    ``per_param_step=False``: one step count for all parameters (one launch); the set of parameters with a gradient must
    not change after the first update.  ``per_param_step=True``: one count per parameter (two launches), like torch.optim:
    the set may change between updates outside CUDA graph capture (the segment table is rebuilt; a graph captured
    earlier keeps its own table), a parameter without a gradient keeps its state and its count, and checkpoints may hold
    differing steps and parameters without state.  In this mode ``step_count`` is the largest per-parameter count, i.e.
    the updates of the parameters that took part in the most of them."""

    def __init__(self, params, kind="adam", lr=1e-3, weight_decay=0, per_param_step=False):
        if kind not in _KINDS:
            raise ValueError("FusedOptimizer kind %r: expected one of %s" % (kind, sorted(_KINDS)))
        if not isinstance(per_param_step, bool):
            raise TypeError("FusedOptimizer per_param_step must be True or False, got %r" % (per_param_step,))
        cls, extra, self.algo = _KINDS[kind]
        self.kind = kind
        self.per_param_step = per_param_step
        # torch's own constructor validates the arguments and gives the exact defaults (= param_groups keys) of this version
        defaults = dict(cls([torch.zeros(1)], lr=lr, weight_decay=weight_decay, **extra).defaults)
        super().__init__(params, defaults)
        plist = self.param_groups[0]["params"]
        for p in plist:
            if not (p.dtype == torch.float32 and p.is_contiguous() and p.device == plist[0].device):
                raise ValueError("FusedOptimizer needs contiguous float32 parameters on one device")
        dev = plist[0].device
        self._hyper = torch.zeros(6, dtype=torch.float64, device=dev)     # LfOptimHyper
        self._counters = torch.zeros(3, dtype=torch.int64, device=dev)    # LfOptimState: step, skipped, ticket
        # per_param_step: the count of parameter i (its slot) whatever tables are built over it
        self._steps = torch.zeros(len(plist), dtype=torch.int64, device=dev) if per_param_step else None
        self._hyper_host = None
        self._table_key = None
        self._captured_tables = []
        self._started = False
        self._hyper_values(self.param_groups[0])

    def add_param_group(self, param_group):
        if self.param_groups:
            raise ValueError("FusedOptimizer supports one parameter group")
        super().add_param_group(param_group)

    # -- hyperparameters ------------------------------------------------------------------------------------------------
    def _hyper_values(self, g):
        """LfOptimHyper of a parameter group; ValueError for a setting the kernel does not implement."""
        for f in _UNSUPPORTED:
            if g.get(f):
                raise ValueError("FusedOptimizer does not implement %s=True" % f)
        if g.get("dampening", 0):
            raise ValueError("FusedOptimizer does not implement dampening")
        if self.kind != "adam" and not g["momentum"] > 0:
            raise ValueError("FusedOptimizer(%r) needs momentum > 0" % self.kind)
        lr, wd = float(g["lr"]), float(g["weight_decay"])
        if self.kind == "adam":
            return (lr, float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]), wd, 0.0)
        if self.kind == "sgd":
            return (lr, 0.0, 0.0, 0.0, wd, float(g["momentum"]))
        return (lr, 0.0, float(g["alpha"]), float(g["eps"]), wd, float(g["momentum"]))

    def sync_hyperparameters(self):
        """Write the device hyperparameter block if a ``param_groups`` value changed on the host (a scheduler's lr).
        Not during capture: a replay reads whatever the block holds then."""
        vals = self._hyper_values(self.param_groups[0])
        if vals != self._hyper_host:
            self._hyper.copy_(torch.tensor(vals, dtype=torch.float64))
            self._hyper_host = vals

    # -- segment table --------------------------------------------------------------------------------------------------
    def grad_params(self):
        return [p for p in self.param_groups[0]["params"] if p.grad is not None]

    def prepare(self, params):
        """Create the state of new parameters and (re)build the device segment table when the gradient pointers changed."""
        key = tuple((p.data_ptr(), p.grad.data_ptr()) for p in params)
        if key == self._table_key:
            return
        _capi.require_cuda(*params)          # the update runs on the kernel only (a CPU optimizer can still load / save)
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("FusedOptimizer: the set of gradients changed during CUDA graph capture")
        with_state = {id(p) for p, st in self.state.items() if st}
        if not self.per_param_step and self._started and with_state != {id(p) for p in params}:
            raise ValueError("FusedOptimizer keeps one step count for all parameters: the set of parameters with a "
                             "gradient must not change after the first update")
        names = STATE_KEYS[self.kind]
        slot = {id(p): i for i, p in enumerate(self.param_groups[0]["params"])}
        rows, chunk = [], 0
        for p in params:
            g = p.grad
            if not (g.dtype == torch.float32 and g.is_contiguous() and g.shape == p.shape and g.device == p.device):
                raise ValueError("FusedOptimizer needs contiguous float32 gradients shaped like their parameters")
            st = self.state[p]
            if not st:
                if self.kind != "sgd":
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                for k in names:
                    st[k] = torch.zeros_like(p, memory_format=torch.contiguous_format)
            s = [st[k] for k in names]
            rows.append([p.data_ptr(), g.data_ptr(), s[0].data_ptr(), s[1].data_ptr() if len(s) > 1 else 0, p.numel(), chunk])
            if self.per_param_step:
                rows[-1].append(slot[id(p)])          # LfOptimSegPP: slot, then reserved (0) in the high word
            chunk += -(-p.numel() // _capi.OPTIM_CHUNK)
        # the previous table is freed here unless a captured graph reads it (launch() keeps those alive)
        self._table = torch.tensor(rows, dtype=torch.int64).to(self._hyper.device)
        self._nsegs, self._nchunks, self._nelem = len(rows), chunk, sum(p.numel() for p in params)
        if self.per_param_step:
            self._slots = (ctypes.c_int * len(rows))(*[r[6] for r in rows])
            self._scalars = torch.empty(len(rows) * _capi.OPTIM_PP_SCALAR_BYTES // 8, dtype=torch.int64,
                                        device=self._hyper.device)
        self._table_key = key

    def launch(self, status=None):
        """The update over the prepared table on the current stream (capturable); ``status``: optional device int32 word,
        nonzero = skip this update."""
        per_elem = 20 if self.kind == "sgd" else 28
        if torch.cuda.is_current_stream_capturing() and not any(t[0] is self._table for t in self._captured_tables):
            # a replay reads them by address for as long as this object lives
            self._captured_tables.append((self._table, self._scalars if self.per_param_step else None))
        if self.per_param_step:
            skipped = ctypes.c_void_p(self._counters.data_ptr() + self._counters.element_size())    # LfOptimState.skipped
            _capi.call("lf_optim_step_pp", self.algo, ptr(self._table), self._slots, self._nsegs, self._nchunks,
                       ptr(self._hyper), ptr(self._steps), self._steps.numel(), ptr(self._scalars), skipped, ptr(status),
                       _capi.stream_ptr(), nbytes=per_elem * self._nelem)
        else:
            _capi.call("lf_optim_step", self.algo, ptr(self._table), self._nsegs, self._nchunks, ptr(self._hyper),
                       ptr(self._counters), ptr(status), _capi.stream_ptr(), nbytes=per_elem * self._nelem)
        self._started = True

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        params = self.grad_params()
        if params:
            self.prepare(params)
            self.sync_hyperparameters()
            self.launch()
            # the kernel writes through raw pointers: bump _version so version-keyed caches (ops_eval) see the update
            torch.autograd.graph.increment_version(params)
        return loss

    # -- counters -------------------------------------------------------------------------------------------------------
    @property
    def step_count(self):
        """Updates applied: the shared count, or with per_param_step the largest per-parameter count."""
        if self.per_param_step:
            return int(self._steps.max().item())
        return int(self._counters[0].item())

    @property
    def step_counts(self):
        """Each parameter's count, in parameter order: torch.optim's per-parameter ``step`` (0 for a parameter never
        updated).  Without per_param_step, the shared count for every parameter that has state."""
        if self.per_param_step:
            return self._steps.tolist()
        step = self.step_count
        return [step if self.state.get(p) else 0 for p in self.param_groups[0]["params"]]

    @property
    def skipped(self):
        return int(self._counters[1].item())

    # -- checkpoints in torch.optim's format ----------------------------------------------------------------------------
    def state_dict(self):
        if self.per_param_step:
            counts = self.step_counts
            for p, n in zip(self.param_groups[0]["params"], counts):
                st = self.state.get(p)
                if st and "step" in st:
                    st["step"] = torch.tensor(float(n), dtype=torch.float32)
            sd = super().state_dict()
            for i, n in enumerate(counts):
                if n == 0:
                    sd["state"].pop(i, None)      # torch.optim holds no state for a parameter before its first update
            return sd
        step = self.step_count
        for st in self.state.values():
            if "step" in st:
                st["step"] = torch.tensor(float(step), dtype=torch.float32)
        sd = super().state_dict()
        if step == 0:
            sd["state"] = {}          # torch.optim holds no state before its first update
        return sd

    def load_state_dict(self, state_dict):
        groups = state_dict["param_groups"]
        if len(groups) != 1:
            raise ValueError("FusedOptimizer supports one parameter group, the state dict has %d" % len(groups))
        self._hyper_values(groups[0])
        names = STATE_KEYS[self.kind]
        steps = {}
        for idx, st in state_dict["state"].items():
            missing = [k for k in names if k not in st]
            if missing:
                raise ValueError("state of parameter %s lacks %s" % (idx, ", ".join(missing)))
            if "step" in st:
                steps[idx] = float(st["step"])
        if self.per_param_step:
            # torch's SGD keeps no step: a momentum buffer means at least one update
            step = 0
            counts = [0] * len(self.param_groups[0]["params"])
            for idx in state_dict["state"]:
                counts[idx] = 1 if self.kind == "sgd" else int(steps.get(idx, 0))
        elif self.kind == "sgd":
            step = 1 if state_dict["state"] else 0
        else:
            if len(set(steps.values())) > 1:
                first = min(steps)
                odd = next(i for i in sorted(steps) if steps[i] != steps[first])
                raise ValueError("parameter %s has step %g but parameter %s has step %g: FusedOptimizer keeps one step "
                                 "count for all parameters" % (odd, steps[odd], first, steps[first]))
            step = int(next(iter(steps.values()))) if steps else 0
        # Existing state tensors keep their addresses: the loaded values are copied into them, so a segment table that a
        # captured graph reads stays valid.  A parameter that has state here but none in the dict would need its own step
        # (per_param_step: it gets one, 0).
        old = {p: [st[k] for k in names] for p, st in self.state.items() if st}
        if step > 0:
            for i, p in enumerate(self.param_groups[0]["params"]):
                if p in old and i not in state_dict["state"]:
                    raise ValueError("parameter %d has optimizer state but none in the state dict: FusedOptimizer keeps one "
                                     "step count for all parameters" % i)
        super().load_state_dict(state_dict)
        replaced = False
        for p, st in self.state.items():
            if not st:
                continue
            for j, k in enumerate(names):
                if p in old:
                    old[p][j].copy_(st[k])
                    st[k] = old[p][j]
                else:         # independent of the caller's tensors (the kernel writes in place)
                    st[k] = st[k].clone(memory_format=torch.contiguous_format)
                    replaced = True
        for p, tensors in old.items():      # no state for p in the dict: fresh zero state
            st = self.state[p]
            if not st:
                if self.kind != "sgd":
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                for k, t in zip(names, tensors):
                    st[k] = t.zero_()
        if self.per_param_step:
            self._steps.copy_(torch.tensor(counts, dtype=torch.int64))
        else:
            self._counters[0].fill_(step)
        if replaced:
            self._table_key = None
        self._hyper_host = None
        self._started = step > 0
