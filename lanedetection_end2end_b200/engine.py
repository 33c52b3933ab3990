"""Whole-step CUDA graph for the training hot path.

One step = zero grads -> ``Net.forward`` -> backprojection loss over the lanes -> backward
(-> flat gradient all-reduce when data-parallel): ~600 kernel launches of a few microseconds
each (SURVEY.md 7.2 #6).  Eagerly, the Python/ctypes cost per launch bounds the step once the kernels
are fast; captured once into a ``torch.cuda.CUDAGraph`` the step is a single replay.  Inputs live
in static device buffers (``copy_`` new batches in, asynchronously from pinned host memory); the loss and
the LSQ status word are static outputs the caller reads when it wants to (no sync inside the step).

The graph only contains our C-ABI kernels, a handful of tiny float64 torch ops of the loss, torch's
graph-safe Philox draws for the Dropout2d masks, and (optionally) the NCCL all-reduce.
"""
import os

import torch

# lf_backproj_loss: one launch for the loss of all lanes + its gradient instead of ~40 tiny float64 torch launches.
# GPU-validated (tests/test_net_gpu.py::test_fused_backprojection_loss_kernel): on by default;
# LANEFIT_FUSED_LOSS=0 falls back to the torch ops of Loss_crit.backprojection_loss.forward_lanes.
FUSED_LOSS = os.environ.get("LANEFIT_FUSED_LOSS", "1") != "0"


def batchnorm_running_stats(model):
    """The running statistics of every BatchNorm container (nn.BatchNorm2d, nn.SyncBatchNorm, ...): a replay updates them
    through raw pointers, so their versions are bumped after it."""
    return [b for m in model.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)
            for b in (m.running_mean, m.running_var) if b is not None]


class GraphedTrainStep:
    """``optimizer``: None (the graph ends with the gradients, the caller steps its optimizer), or an
    ``optim.FusedOptimizer`` over the model's parameters: the graph then starts by zeroing ``model.lsq_status`` (the
    status becomes per-step) and ends, after the reducer, with the update guarded by that word -- a batch with a singular
    system changes no parameter or optimizer state, with no host synchronisation.  With a reducer the guard reads the
    word's maximum over the ranks (one all-reduce of one element, ddp.any_rank_nonzero), so every rank skips or updates
    together and the replicas stay identical.  Each call writes the optimizer's
    hyperparameters first if a param_groups value changed (schedulers work without a recapture)."""

    def __init__(self, model, criterion, nclasses, example_x, example_xgt, example_valid, reducer=None, warmup=3,
                 capture_error_mode="global", extra_loss=None, global_valid=False, optimizer=None):
        if optimizer is not None:
            from .optim import FusedOptimizer
            if not isinstance(optimizer, FusedOptimizer):
                raise TypeError("GraphedTrainStep captures the update of an optim.FusedOptimizer only, got %s"
                                % type(optimizer).__name__)
        self.optimizer = optimizer
        self.model = model
        self.global_valid = global_valid  # batch-global sum(valid) normaliser across ranks (ddp.lane_valid_scale)
        self.extra_loss = extra_loss      # callable(forward 9-tuple) -> scalar added to the loss (e.g. the --clas head losses)
        self.crit = criterion
        self.L = nclasses
        self.reducer = reducer
        dev = example_x.device
        self.x = example_x.clone()
        self.xgt = example_xgt.clone()
        self.valid = example_valid.clone()
        self.gt_line = torch.zeros(example_x.shape[0], 4)
        model.defer_status_check = True
        self.params = [p for p in model.parameters() if p.requires_grad]

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):
                self._eager_step(first=True)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        # gradients now exist as persistent tensors; the captured step zeroes and re-accumulates them
        if reducer is not None and hasattr(reducer, "attach"):
            reducer.attach()          # gradients become views of the flat all-reduce buffer: no pack / unpack copies
        self.grads = [p.grad for p in self.params if p.grad is not None]
        if optimizer is not None:
            self.updated = optimizer.grad_params()
            optimizer.prepare(self.updated)          # state and segment table exist before the capture
            optimizer.sync_hyperparameters()
            self.skip_word = torch.zeros(1, dtype=torch.int32, device=dev)   # status word reduced over the ranks
            # what a replay writes through raw pointers besides the parameters: the BatchNorm running statistics
            self.written = self.updated + batchnorm_running_stats(model)
        self.graph = torch.cuda.CUDAGraph()
        # with NCCL in the graph use capture_error_mode="thread_local": the process group's watchdog thread polls CUDA
        # events, which the default "global" mode treats as a capture violation
        with torch.cuda.graph(self.graph, capture_error_mode=capture_error_mode):
            self.loss = self._eager_step(first=False)
        self.status = model.lsq_status

    def _eager_step(self, first):
        if first:
            self.model.zero_grad(set_to_none=True)
        else:
            if self.optimizer is not None:
                self.model.lsq_status.zero_()
            torch._foreach_zero_(self.grads)
        out = self.model(self.x, self.gt_line, True)
        scale = None
        if self.global_valid:
            from .ddp import lane_valid_scale
            scale = lane_valid_scale(self.valid, self.L)
        if FUSED_LOSS and hasattr(self.crit, "_fused_host_constants"):
            from .Loss_crit import fused_backprojection_loss
            loss, _ = fused_backprojection_loss(self.crit, out[:self.L], self.xgt, self.valid, lane_scale=scale)
        elif hasattr(self.crit, "forward_lanes"):
            loss, _ = self.crit.forward_lanes(out[:self.L], self.xgt, self.valid, lane_scale=scale)    # all lanes in one pass
        else:
            loss = 0
            for l in range(self.L):
                ll, _ = self.crit(out[l], self.xgt[:, l], self.valid[:, l])
                loss = loss + ll
            loss = loss / self.L
        if self.extra_loss is not None:
            loss = loss + self.extra_loss(out)
        loss.backward()
        if self.reducer is not None:
            self.reducer()
        if not first and self.optimizer is not None:
            status = self.model.lsq_status
            if self.reducer is not None:
                # data-parallel: the ranks share the averaged gradients, so a singular system on any rank skips every rank
                from .ddp import any_rank_nonzero
                status = any_rank_nonzero(status, self.skip_word, getattr(self.reducer, "group", None))
            self.optimizer.launch(status=status)
        return loss.detach()

    def load(self, x, xgt, valid):
        """Stage a new batch (device or pinned-host tensors) into the static input buffers."""
        self.x.copy_(x, non_blocking=True)
        self.xgt.copy_(xgt, non_blocking=True)
        self.valid.copy_(valid, non_blocking=True)

    # -- double-buffered input pipeline: the H2D copy of batch i+1 runs on a copy stream while step i computes
    def prefetch(self, x, xgt, valid):
        """Start copying the NEXT batch (pinned host tensors) into the staging buffers on the copy stream."""
        if not hasattr(self, "_copy_stream"):
            dev = self.x.device
            self._copy_stream = torch.cuda.Stream(device=dev)
            self._stage = [torch.empty_like(self.x), torch.empty_like(self.xgt), torch.empty_like(self.valid)]
            self._ready = torch.cuda.Event()
            self._consumed = torch.cuda.Event()
            self._consumed.record(torch.cuda.current_stream(dev))
        self._copy_stream.wait_event(self._consumed)     # staging buffers were drained by swap_in()
        with torch.cuda.stream(self._copy_stream):
            for dst, src in zip(self._stage, (x, xgt, valid)):
                dst.copy_(src, non_blocking=True)
            self._ready.record(self._copy_stream)

    def swap_in(self):
        """Move the prefetched batch into the graph's static inputs (device-to-device, on the compute stream)."""
        cur = torch.cuda.current_stream(self.x.device)
        cur.wait_event(self._ready)
        self.x.copy_(self._stage[0], non_blocking=True)
        self.xgt.copy_(self._stage[1], non_blocking=True)
        self.valid.copy_(self._stage[2], non_blocking=True)
        self._consumed.record(cur)

    def __call__(self):
        if self.optimizer is None:
            self.graph.replay()
            return self.loss
        self.optimizer.sync_hyperparameters()
        self.graph.replay()
        torch.autograd.graph.increment_version(self.written)    # version-keyed caches (ops_eval) see the update
        return self.loss


class GraphedInference:
    """Eval-mode forward (BatchNorm-folded launches, ops_eval.py) captured once into a CUDA graph and replayed per batch:
    what the reference's validate() / test_model() loops do per batch (BP/main.py:452, BP/test.py:53-55), without the ~25 us
    of ctypes / Python per launch.  ``infer(x)`` copies the batch into the static input and replays; the returned 9-tuple
    (beta0..3, masked, output, line, horizon, output_seg) aliases static buffers that the next call overwrites.
    ``model.lsq_status`` (device int32, OR-ed) reports singular systems; `check()` reads it (one sync)."""

    def __init__(self, model, example_x, warmup=2):
        self.model = model.eval()
        model.defer_status_check = True
        self.x = example_x.clone()
        self.gt_line = torch.zeros(example_x.shape[0], 4)
        dev = example_x.device
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(max(1, warmup)):             # builds and caches the folded operands outside the capture
                model(self.x, self.gt_line, True)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(self.graph):
            self.out = model(self.x, self.gt_line, True)

    def infer(self, x):
        self.x.copy_(x, non_blocking=True)
        self.graph.replay()
        return self.out

    def check(self):
        st = int(self.model.lsq_status.item())
        if st:
            self.model.lsq_status.zero_()
            raise RuntimeError("status word %d (1 singular / 2 non-finite / 4 not positive definite normal matrix)" % st)
