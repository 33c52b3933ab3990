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
import time

import torch


def model_forward(model, x, gt_line, end_to_end):
    """Net.forward of either experiment: the back-projection Net takes (input, gt_line, end_to_end), the bird's-eye-view
    Net (``takes_gt_line = False``) takes (input, end_to_end)."""
    if getattr(model, "takes_gt_line", True):
        return model(x, gt_line, end_to_end)
    return model(x, end_to_end)


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
    hyperparameters first if a param_groups value changed (schedulers work without a recapture).  An optimizer with
    ``max_grad_norm`` takes the gradients' norm after the reducer, so under data parallelism every rank clips by the same
    coefficient and a non-finite gradient skips every rank's update.

    ``gt_line``: optional example [B, 4] tensor, cloned into a static buffer ``self.gt_line`` that the forward reads (the
    segmentation branch's substitution, end_to_end=False); default a host tensor of zeros.  The loss is
    Loss_crit.fused_backprojection_loss of ``criterion`` (a Loss_crit.backprojection_loss) over the ``nclasses`` lanes,
    plus ``extra_loss``; ``loss_fn``: optional callable(forward 9-tuple) -> scalar loss that replaces both.  ``post``:
    optional callable(forward 9-tuple, detached loss) run at the end of every step, after the update (its return value is
    ``self.post_out``); the warm-up steps run it too.

    ``early_return=True``: the forward is ``model(x, gt_line, end_to_end, early_return=True)``, the decoder output alone
    (the segmentation pretraining of --pretrained, BP/main.py:255-258), which ``loss_fn`` and ``post`` then receive in
    place of the 9-tuple.  Without the least-squares layer no batch can be singular: the update runs unguarded."""

    def __init__(self, model, criterion, nclasses, example_x, example_xgt, example_valid, reducer=None, warmup=3,
                 capture_error_mode="global", extra_loss=None, global_valid=False, optimizer=None, gt_line=None,
                 end_to_end=True, loss_fn=None, post=None, early_return=False):
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
        self.gt_line = torch.zeros(example_x.shape[0], 4) if gt_line is None else gt_line.clone()
        self.end_to_end = end_to_end
        self.early_return = early_return
        self.loss_fn = loss_fn
        self.post = post
        self.post_out = None
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
            if self.optimizer is not None and not self.early_return:
                self.model.lsq_status.zero_()
            torch._foreach_zero_(self.grads)
        if self.early_return:
            out = self.model(self.x, self.gt_line, self.end_to_end, early_return=True)
        else:
            out = model_forward(self.model, self.x, self.gt_line, self.end_to_end)
        scale = None
        if self.global_valid:
            from .ddp import lane_valid_scale
            scale = lane_valid_scale(self.valid, self.L)
        if self.loss_fn is not None:
            loss = self.loss_fn(out)
        else:
            from .Loss_crit import fused_backprojection_loss
            loss, _ = fused_backprojection_loss(self.crit, out[:self.L], self.xgt, self.valid, lane_scale=scale)
            if self.extra_loss is not None:
                loss = loss + self.extra_loss(out)
        loss.backward()
        if self.reducer is not None:
            self.reducer()
        if not first and self.optimizer is not None:
            status = None if self.early_return else self.model.lsq_status
            if self.reducer is not None and status is not None:
                # data-parallel: the ranks share the averaged gradients, so a singular system on any rank skips every rank
                from .ddp import any_rank_nonzero
                status = any_rank_nonzero(status, self.skip_word, getattr(self.reducer, "group", None))
            self.optimizer.launch(status=status)
        loss = loss.detach()
        if self.post is not None:
            self.post_out = self.post(out, loss)
        return loss

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
    ``model.lsq_status`` (device int32, OR-ed) reports singular systems; `check()` reads it (one sync).
    ``post``: optional callable(9-tuple) captured right after the forward (and run by every warm-up pass); its return value
    is ``self.post_out``, static like ``self.out``.
    ``gt_line`` (optional example [B, 4] tensor, cloned into the static ``self.gt_line``) and ``end_to_end`` are the
    forward's arguments; by default host zeros and True."""

    def __init__(self, model, example_x, warmup=2, post=None, gt_line=None, end_to_end=True):
        self.model = model.eval()
        model.defer_status_check = True
        self.x = example_x.clone()
        self.gt_line = torch.zeros(example_x.shape[0], 4) if gt_line is None else gt_line.clone()
        self.post_out = None
        dev = example_x.device
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(max(1, warmup)):             # builds and caches the folded operands outside the capture
                out = model_forward(model, self.x, self.gt_line, end_to_end)
                if post is not None:
                    post(out)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.no_grad(), torch.cuda.graph(self.graph):
            self.out = model_forward(model, self.x, self.gt_line, end_to_end)
            if post is not None:
                self.post_out = post(self.out)

    def infer(self, x):
        self.x.copy_(x, non_blocking=True)
        self.graph.replay()
        return self.out

    def check(self):
        st = int(self.model.lsq_status.item())
        if st:
            self.model.lsq_status.zero_()
            raise RuntimeError("status word %d (1 singular / 2 non-finite / 4 not positive definite normal matrix)" % st)


class DeviceMeters:
    """The reference's AverageMeters (BP/Networks/utils.py AverageMeter) on the device: one float64 (val, sum, count) row per
    name, updated as ``sum += val * n; count += n`` -- AverageMeter.update's Python-float arithmetic -- so the averages come
    out bit for bit.  ``update`` is guarded by a device bool (no synchronisation, capturable); ``read`` is one copy."""

    def __init__(self, names, device):
        self.names = list(names)
        self.t = torch.zeros(len(self.names), 3, dtype=torch.float64, device=device)

    def update(self, name, val, ok, n=1):
        row = self.t[self.names.index(name)]
        v = val.detach().reshape(()).double()
        row[0].copy_(torch.where(ok, v, row[0]))
        row[1].add_(torch.where(ok, v * n, 0.0))
        row[2].add_(ok.double() * n)

    def read(self):
        """name -> (val, avg) as AverageMeter holds them (0, 0 before the first update)."""
        return {k: (v, s / c) if c else (0, 0) for k, (v, s, c) in zip(self.names, self.t.tolist())}


class BatchStatus:
    """A device log of each batch's LSQ status word: ``record`` (capturable) appends ``status`` at a device position and
    zeroes it for the next batch.  ``skipped`` reads it once: the host labels of the batches whose word was nonzero."""

    def __init__(self, capacity, device):
        self.log = torch.zeros(max(1, capacity), dtype=torch.int32, device=device)
        self.pos = torch.zeros(1, dtype=torch.int64, device=device)

    def check(self, i):
        if i >= self.log.numel():
            raise ValueError("the loader yielded more batches than its len() of %d" % self.log.numel())

    def record(self, status):
        self.log.index_copy_(0, self.pos, status.reshape(1))
        self.pos.add_(1)

    def print_skipped(self, labels):
        """The reference's line for each skipped batch, in order (BP/main.py:289-292: the batch's idx, then the error)."""
        from .ops_lsq import status_message
        for st, idx in zip(self.log[:len(labels)].tolist(), labels):
            if st:
                print("Batch with idx {} skipped due to singular matrix".format(idx.numpy()))
                print(status_message(st))


def lane_losses(criterion, out, lanes, vp, L):
    """The lane loop of BP/main.py:296-305 (and :309-317, :460-469) with its ops in its order: the mean over lanes of the
    per-lane criterion calls, and the four x_cal (None past L lanes)."""
    x_cal2 = x_cal3 = None
    loss_left, x_cal0 = criterion(out[0], lanes[:, 0, :], vp[:, 0])
    loss_right, x_cal1 = criterion(out[1], lanes[:, 1, :], vp[:, 1])
    if L > 3:
        loss_left1, x_cal2 = criterion(out[2], lanes[:, 2, :], vp[:, 2])
        loss_right1, x_cal3 = criterion(out[3], lanes[:, 3, :], vp[:, 3])
        loss_left += loss_left1
        loss_right += loss_right1
    return (loss_left + loss_right) / L, [x_cal0, x_cal1, x_cal2, x_cal3]


def _reporting(i, freq):
    return freq > 0 and (i + 1) % freq == 0


def _keeping_batchnorm_stats(model, build):
    """``build()`` with the BatchNorm running statistics restored afterwards: a GraphedTrainStep's warm-up steps are
    training forwards, which would move them."""
    bns = [m for m in model.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)]
    saved = [[t.clone() if t is not None else None for t in (m.running_mean, m.running_var, m.num_batches_tracked)]
             for m in bns]
    out = build()
    for m, ts in zip(bns, saved):
        for t, v in zip((m.running_mean, m.running_var, m.num_batches_tracked), ts):
            if t is not None:
                t.copy_(v)
    return out


def _device_copies(tensors, casts, dev):
    """Static device buffers for a batch: clones of ``tensors`` (name -> tensor), then ``casts`` (name -> dtype)."""
    st = {k: v.to(dev, non_blocking=True).clone() for k, v in tensors.items()}
    st.update({k: st[k].to(dtype) for k, dtype in casts.items()})
    return st


def _train_replays(loader, model, optimizer, static, fields, casts, post, report=None, print_freq=0, save_freq=0,
                   gt_line=False, early_return=False, **step_kw):
    """The loop of the graphed training epochs: each batch one replay of a GraphedTrainStep over the FusedOptimizer
    ``optimizer``.  Returns the step, None when the loader yields no batch.

    ``fields(batch)`` names the loader tuple's tensors that become static device buffers: ``static`` receives the first
    batch's copies (_device_copies with ``casts``), later batches are copied into them, and every batch must have the
    first one's size.  ``static["input"]`` (with ``gt_line=True`` also ``static["gt_line"]``, which the forward then
    reads) is the step's own buffer.  ``step_kw`` (loss_fn, end_to_end) and ``early_return`` go to the GraphedTrainStep;
    the loss reads its batch through loss_fn.  ``post(out, loss)`` runs in the captured step only, not in the warm-up
    steps; after it the step's LSQ status word is logged (not with ``early_return``, which has no least-squares layer),
    and the reference's line for each skipped batch is printed at the end.  ``report(i, printing, saving, batch,
    post_out, (batch time, its average))`` runs at the print_freq / save_freq points of a batch that was not skipped:
    the only host synchronisations before the end.  With gradient clipping on (``optimizer.max_grad_norm``), one line at
    the end reports the updates that a non-finite gradient skipped during the epoch, if any."""
    dev = next(model.parameters()).device
    model.train()
    status = None if early_return else BatchStatus(len(loader), dev)
    # a device copy of LfGradClip.nonfinite_skipped: reading the count here would add a synchronisation
    nonfinite0 = None if optimizer.max_grad_norm is None else optimizer._clip[2].clone()

    def captured_post(out, loss):
        if not torch.cuda.is_current_stream_capturing():
            return None                      # warm-up steps: no meter or log entry
        ret = post(out, loss)
        if status is not None:
            status.record(model.lsq_status)
        return ret

    step, labels = None, []
    bt_sum, bt_n, end = 0.0, 0, time.time()
    deferred = model.defer_status_check
    try:
        for i, batch in enumerate(loader):
            tensors = fields(batch)
            if step is None:
                static.update(_device_copies(tensors, casts, dev))
                none = torch.empty(0, device=dev)
                step = _keeping_batchnorm_stats(model, lambda: GraphedTrainStep(
                    model, None, 0, static["input"], none, none, optimizer=optimizer,
                    gt_line=static["gt_line"] if gt_line else None, post=captured_post, early_return=early_return,
                    **step_kw))
                static["input"] = step.x              # the step's own copies are what its forward reads
                if gt_line:
                    static["gt_line"] = step.gt_line
            else:
                if batch[0].shape[0] != step.x.shape[0]:
                    raise ValueError("batch of %d images after a first batch of %d: a training epoch replays one batch "
                                     "size" % (batch[0].shape[0], step.x.shape[0]))
                for k, v in tensors.items():
                    static[k].copy_(v, non_blocking=True)
            if status is not None:
                status.check(i)
            labels.append(batch[3])
            step()
            now = time.time()
            bt_val, end = now - end, now
            bt_sum, bt_n = bt_sum + bt_val, bt_n + 1
            printing, saving = _reporting(i, print_freq), _reporting(i, save_freq)
            # a skipped batch reports nothing, as main.py's `continue`
            if (printing or saving) and not int(status.log[i]):
                report(i, printing, saving, batch, step.post_out, (bt_val, bt_sum / bt_n))
    finally:
        model.defer_status_check = deferred
    if status is not None:
        status.print_skipped(labels)
    if nonfinite0 is not None:
        n = int((optimizer._clip[2] - nonfinite0).item())
        if n:
            print("%d of %d updates skipped: non-finite gradients" % (n, len(labels)))
    return step


def _valid_replays(loader, model, fields, casts, post, report, print_freq, gt_line=False, end_to_end=True):
    """The loop of the graphed validation passes: each batch one replay of a GraphedInference, with one graph and one
    set of static buffers per batch size (a batch shorter than the first gets its own; a larger one raises ValueError).

    ``fields`` and ``casts`` as in _train_replays, per graph; with ``gt_line=True`` the forward reads the graph's
    ``st["gt_line"]``.  ``post(out, st)`` is the graph's post on its static batch ``st``; after it the captured pass
    logs and zeroes the LSQ status word, and the reference's line for each skipped batch is printed at the end.
    ``report(i, printing, saving, batch, graph, st)`` runs at the print_freq / 25 points of a batch that was not
    skipped: the only host synchronisations before the end."""
    dev = next(model.parameters()).device
    status = BatchStatus(len(loader), dev)
    graphs = {}                     # rows -> (GraphedInference, static batch tensors)

    def build(tensors):
        st = _device_copies(tensors, casts, dev)

        def captured_post(out):
            ret = post(out, st)
            if torch.cuda.is_current_stream_capturing():
                status.record(model.lsq_status)
                model.lsq_status.zero_()
            return ret

        g = GraphedInference(model, st["input"], post=captured_post, gt_line=st["gt_line"] if gt_line else None,
                             end_to_end=end_to_end)
        st["input"] = g.x
        if gt_line:
            st["gt_line"] = g.gt_line        # the forward's substitution and the accuracies read one buffer
        model.lsq_status.zero_()
        return g, st

    first, labels = None, []
    deferred = model.defer_status_check
    try:
        with torch.no_grad():
            for i, batch in enumerate(loader):
                tensors, n = fields(batch), batch[0].shape[0]
                status.check(i)
                if first is None:
                    first = n
                elif n > first:
                    raise ValueError("batch of %d images after a first batch of %d" % (n, first))
                if n in graphs:
                    g, st = graphs[n]
                    for k, v in tensors.items():
                        st[k].copy_(v, non_blocking=True)
                else:
                    g, st = graphs[n] = build(tensors)
                labels.append(batch[3])
                g.graph.replay()
                printing, saving = _reporting(i, print_freq), _reporting(i, 25)
                # a skipped batch reports nothing, as main.py's `continue`
                if (printing or saving) and not int(status.log[i]):
                    report(i, printing, saving, batch, g, st)
    finally:
        model.defer_status_check = deferred
    status.print_skipped(labels)


def check_lane_curriculum(args):
    """--lane_curriculum E: ValueError unless E == 0 (off) or E > 0 with 4 lanes."""
    e = getattr(args, "lane_curriculum", 0)
    if e < 0:
        raise ValueError("--lane_curriculum takes a number of epochs >= 0, got %d" % e)
    if e > 0 and args.nclasses != 4:
        raise ValueError("--lane_curriculum fits the egolanes first and then all four lanes: it needs --nclasses 4, got "
                         "%d" % args.nclasses)


def curriculum_lanes(args, epoch):
    """The lanes an end-to-end training epoch fits under --lane_curriculum E: lanes 0 and 1 (the egolanes, in the loader's
    lane order) before epoch E, None (every lane) from E on and whenever the flag is off."""
    e = getattr(args, "lane_curriculum", 0)
    return 2 if e > 0 and epoch < e else None


class _FitLanes:
    """``with _FitLanes(model, K):`` sets ``model.fit_lanes`` to K and restores the previous value on exit."""

    def __init__(self, model, lanes):
        self.model, self.lanes = model, lanes

    def __enter__(self):
        self.saved = getattr(self.model, "fit_lanes", None)
        self.model.fit_lanes = self.lanes

    def __exit__(self, *exc):
        self.model.fit_lanes = self.saved


def check_bp_args(args, criterion, model):
    """The settings train_epoch and inference.validate run: ValueError naming the first one they do not.  A criterion
    built with --learn_homography is bound to ``model``'s learned warp."""
    check_lane_curriculum(args)
    if args.clas and not args.end_to_end:
        raise ValueError("--clas needs --end_to_end True (the heads run on the end-to-end branch only)")
    if not args.end_to_end and args.nclasses != 4:
        raise ValueError("--end_to_end False needs 4 lanes: the reference's gt_line substitution does not broadcast the "
                         "loader's 4 line flags over %d lane maps" % args.nclasses)
    if getattr(criterion, "learn_homography", False):
        criterion.bind(model)


def train_epoch(loader, model, optimizer, criterion, criterion_seg, criterion_line_class, criterion_horizon, args, epoch,
                seg_metrics=None):
    """One training epoch of the reference's main.py loop (BP/main.py:225-359), each batch one replay of a
    GraphedTrainStep that holds the forward, the loss, the backward, the fused optimizer's update and the meter updates.
    Returns (losses.avg, rmse_metric.avg) -- rmse_metric is updated with --end_to_end False only, as in the reference.

    The loader yields the train loader's 7-tuples (input, gt, lanes, idx, gt_line, gt_horizon, valid_points), on the
    device as Dataloader.Load_Data_new gives them (host tensors are copied in); every batch has the first one's size (the
    train loader drops its last batch).  ``optimizer`` must be an optim.FusedOptimizer (define_optim(..., fused=True)): the
    update sits in the graph, guarded by the LSQ status word, so a batch with a singular system changes no parameter, no
    optimizer state and no meter, without a host synchronisation; the reference's line for each such batch is printed at the
    end of the epoch.  The host synchronises only at the print_freq lines, at save_weightmap('train', ...) every save_freq
    batches and at the end.

    Loss: end-to-end, the fused lf_backproj_loss (Loss_crit.fused_backprojection_loss), whose lane sum is reassociated
    against main.py:296-305's per-lane criterion calls (equal to about 1e-12 relative); with --clas, ``loss * weight_fit +
    (bce_line.double() + bce_horizon.double()) * weight_class``.  --end_to_end False: criterion_seg(output, gt), with the
    least-squares fit and the rmse metric computed without gradient (main.py:306-318).  clip_grad_norm is accepted and does
    nothing: main.py:334-335 clips the gradients of the previous batch before zero_grad() discards them, so it never changes
    an update.  Clipping is asked for on the optimizer instead (define_optim(..., fused=True, max_grad_norm=...)): the
    update then scales the gradients by torch's clip_grad_norm_ coefficient, and an update that a non-finite gradient
    skipped is reported in one line at the end of the epoch.  Dropout masks are drawn in the graph from torch's
    graph-safe Philox offsets; they do not repeat an eager run's masks.  BatchNorm running statistics are those of the epoch's batches (the capture's warm-up steps leave them as
    they were).

    --pretrained needs a FusedOptimizer built with per_param_step=True (define_optim(..., fused=True,
    per_param_step=True)), since its phases train different parameter sets; otherwise it raises ValueError.  The phase
    comes from ``epoch`` and ``args`` as main.py's get_flags gives it (``args`` is not changed): a skip epoch (epoch <
    skip_epochs and < pretrain_epochs) replays ``model(input, gt_line, False, early_return=True)`` -- the decoder through
    output_conv2, no least-squares layer -- with the loss criterion_seg(output, gt) and the update unguarded
    (main.py:255-282), and returns (losses_skip.avg, 0.0); main.py prints no per-batch line there, and its plot at
    save_freq is not drawn.  Every other epoch follows ``args.end_to_end``, which the caller's get_flags(epoch) sets:
    the segmentation branch through output_conv2, or end to end through output_conv and the heads, whose optimizer
    state starts at step 1 while output_conv2 keeps its state.  --clas with --end_to_end False raises ValueError outside
    the skip epochs (main.py:320-325 would call the line criterion on None).

    A model built with --seg_proxy (``model.seg_proxy``) trains its second decoder in the same step: the loss is
    Loss_crit.seg_proxy_loss, ``L_fit + weight_seg_proxy * criterion_seg(output_seg, gt)`` in float64, L_fit the loss
    above; losses.avg is that total.  The proxy term has a device meter of its own; pass a dict as ``seg_metrics`` to
    receive its average under "ce".

    --lane_curriculum E (4 lanes): an end-to-end epoch < E sets ``model.fit_lanes = 2`` for its replays (restored on
    exit), so the fit, the status word that guards the update and the loss cover the egolanes only: the loss is
    fused_backprojection_loss over lanes 0 and 1, the 2-lane model's, while the --clas heads keep their 4-lane losses.
    From epoch E on every lane is fitted, as without the flag.  With weight_decay > 0 the optimizer still decays the
    outer lanes' output_conv channels in those epochs, whose gradient is zero."""
    from .optim import FusedOptimizer
    from .Loss_crit import fused_backprojection_loss, seg_proxy_loss
    from .Networks import utils as nutils
    if not isinstance(optimizer, FusedOptimizer):
        raise TypeError("train_epoch runs the update in the graph: it needs an optim.FusedOptimizer "
                        "(define_optim(..., fused=True)), got %s" % type(optimizer).__name__)
    if args.pretrained and not optimizer.per_param_step:
        raise ValueError("train_epoch runs --pretrained with a per-parameter step count only: its segmentation phase and "
                         "the switch to end-to-end change the parameter set.  Build the optimizer with "
                         "define_optim(..., fused=True, per_param_step=True)")
    if args.pretrained and epoch < args.pretrain_epochs and epoch < args.skip_epochs:
        return _train_skip_epoch(loader, model, optimizer, criterion_seg)
    check_bp_args(args, criterion, model)
    e2e, L = bool(args.end_to_end), args.nclasses
    proxy = bool(getattr(model, "seg_proxy", False))
    meters = DeviceMeters(("loss", "rmse") + (("seg_proxy",) if proxy else ()), next(model.parameters()).device)
    static = {}

    # --lane_curriculum: an end-to-end epoch before E fits (and takes the loss over) the egolanes only
    K = (curriculum_lanes(args, epoch) if e2e else None) or L

    def loss_fn(out):
        if not e2e:
            with torch.no_grad():
                static["rmse"], static["x_cal"] = lane_losses(criterion, out, static["lanes"], static["valid"], L)
            return criterion_seg(out[5], static["gt"])
        loss, x_cal = fused_backprojection_loss(criterion, out[:K], static["lanes"], static["valid"])
        static["x_cal"] = [x_cal[:, l] for l in range(K)] + [None] * (4 - K)
        if args.clas:
            loss_horizon = criterion_horizon(out[7], static["gt_horizon"]).double()
            loss_line = criterion_line_class(out[6], static["gt_line"]).double()
            loss = loss * args.weight_fit + (loss_line + loss_horizon) * args.weight_class
        if proxy:
            loss, static["seg_proxy"] = seg_proxy_loss(loss, criterion_seg, out[8], static["gt"], args.weight_seg_proxy)
        return loss

    def post(out, loss):
        ok = model.lsq_status.reshape(()).eq(0)
        n = static["input"].shape[0]
        if not e2e:
            meters.update("rmse", static["rmse"], ok, n)
        meters.update("loss", loss, ok, n)
        if proxy:
            meters.update("seg_proxy", static["seg_proxy"], ok, n)
        return out[4]

    def report(i, printing, saving, batch, masked, bt):
        if printing:
            m = meters.read()
            print('Epoch: [{0}][{1}/{2}]\t'
                  'Time {3:.3f} ({4:.3f})\t'
                  'Loss {loss[0]:.8f} ({loss[1]:.8f})\t'
                  'rmse_metric {rmse[0]:.8f} ({rmse[1]:.8f})'.format(
                      epoch + 1, i + 1, len(loader), bt[0], bt[1], loss=m["loss"], rmse=m["rmse"]))
        if saving:
            lanes = static["lanes"]
            nutils.save_weightmap('train', masked, *static["x_cal"], lanes[:, 0, :], lanes[:, 1, :], lanes[:, 2, :],
                                  lanes[:, 3, :], static["gt"], 0, i, static["input"], args.no_ortho, args.resize,
                                  args.save_path, K, args.no_mapping)

    fields = lambda b: {"input": b[0], "gt": b[1].squeeze(1), "lanes": b[2], "gt_line": b[4], "gt_horizon": b[5],
                        "valid": b[6]}
    casts = {"input": torch.float32, "gt": torch.int64}
    with _FitLanes(model, K if K < L else None):
        step = _train_replays(loader, model, optimizer, static, fields, casts, post, report, args.print_freq,
                              args.save_freq, gt_line=not e2e, loss_fn=loss_fn, end_to_end=e2e)
    if step is None:
        return 0, 0
    m = meters.read()
    if proxy and seg_metrics is not None:
        seg_metrics["ce"] = m["seg_proxy"][1]
    return m["loss"][1], m["rmse"][1]


def _train_skip_epoch(loader, model, optimizer, criterion_seg):
    """A skip epoch of --pretrained (BP/main.py:255-282) as graph replays: the decoder output through output_conv2, the
    segmentation loss and the unguarded update; returns (losses_skip.avg, 0.0)."""
    dev = next(model.parameters()).device
    meters = DeviceMeters(("loss_skip",), dev)
    always = torch.ones((), dtype=torch.bool, device=dev)
    static = {}

    def post(out, loss):
        meters.update("loss_skip", loss, always, static["input"].shape[0])

    if _train_replays(loader, model, optimizer, static, lambda b: {"input": b[0], "gt": b[1].squeeze(1)},
                      {"input": torch.float32, "gt": torch.int64}, post, early_return=True, end_to_end=False,
                      loss_fn=lambda out: criterion_seg(out, static["gt"])) is None:
        return 0, 0
    return meters.read()["loss_skip"][1], 0.0


def check_bev_args(args):
    """The settings train_epoch_bev and inference.validate_bev run: ValueError naming the first one they do not."""
    from .Loss_crit import AREA_WEIGHTS
    check_lane_curriculum(args)
    if args.clas and (args.nclasses != 4 or not args.end_to_end):
        raise ValueError("--clas needs 4 lanes and --end_to_end True (BEV/main.py:39-40; the heads run on the end-to-end "
                         "branch only), got %d lanes with end_to_end %s" % (args.nclasses, bool(args.end_to_end)))
    if args.pretrained:
        raise ValueError("--pretrained is not supported: its segmentation phase and the switch to end-to-end change the "
                         "parameter set, which a FusedOptimizer refuses")
    if args.loss_policy != "area":
        raise ValueError("loss_policy %r is not supported: the bird's-eye-view loop runs the area loss" % args.loss_policy)
    if args.order != 2:
        raise ValueError("order %d is not supported: the area loss and the exact-area metric take order 2 (three "
                         "coefficients, as the loader's params)" % args.order)
    if args.weight_funct not in AREA_WEIGHTS:
        raise ValueError("unknown weight_funct %r (none, linear or quadratic)" % (args.weight_funct,))
    if not args.end_to_end and args.nclasses != 2:
        raise ValueError("--end_to_end False needs 2 lanes: the bird's-eye-view Net's segmentation branch fits two lane "
                         "maps")


def clas_loss(loss, out, st, criterion_line_class, criterion_horizon, args):
    """BEV/main.py:250-253 (and :429-431): the fit loss combined with the line-type and horizon heads' losses, float32."""
    loss_horizon = criterion_horizon(out[8], st["gt_horizon"])
    loss_line = criterion_line_class(out[7], st["gt_line"])
    return loss * args.weight_fit + (loss_line + loss_horizon) * args.weight_class


def train_epoch_bev(loader, model, optimizer, criterion, criterion_seg, criterion_line_class, criterion_horizon, args, epoch):
    """One training epoch of the bird's-eye-view experiment's main.py loop (Birds_Eye_View_Loss/main.py:186-295), each
    batch one replay of a GraphedTrainStep that holds the forward, the loss, the backward, the fused optimizer's update
    and the meter updates.  Returns (losses.avg, avg_area.avg, exact_area.avg).

    The loader yields the BEV train loader's 6-tuples (input, gt, params, idx, gt_line, gt_horizon), on the device as
    bev.Dataloader.Load_Data_new gives them (host tensors are copied in); every batch has the first one's size.
    ``optimizer`` must be an optim.FusedOptimizer: the update sits in the graph, guarded by the LSQ status word, so a batch
    with a singular system changes no parameter, no optimizer state and no meter, without a host synchronisation; the
    reference's line for each such batch is printed at the end of the epoch.  The host synchronises only at the print_freq
    lines, at save_weightmap('train', ...) every save_freq batches and at the end.

    End-to-end, the loss is Loss_crit.fused_area_loss over the lanes (main.py:222-237; the 4-lane masks change nothing,
    see there): float64 terms rounded once, so it equals the reference's float32 sum to rounding.  --end_to_end False:
    criterion_seg(output, gt), and the 2-lane area without gradient as avg_area (main.py:239-244).  The exact-area metric
    (main.py:272-280) comes from the same launch, per image bit-identical to the reference's CPU polynomial.  With --clas
    (4 lanes, end to end) the loss is ``loss * weight_fit + (loss_line + loss_horizon) * weight_class`` in float32, as
    main.py:246-253 forms it before losses.update: criterion_line_class on the line head's [B, 3, 4] logits against the
    loader's gt_line, criterion_horizon on the horizon head against gt_horizon.  --clas with other lane counts or
    --end_to_end False, --pretrained, loss policies other than area, orders other than 2 and other lane counts raise
    ValueError (check_bev_args).  clip_grad_norm is accepted and does nothing, as in train_epoch; clipping is asked
    for on the optimizer (max_grad_norm), as there.  Dropout masks are drawn in the
    graph; BatchNorm running statistics are those of the epoch's batches.  --lane_curriculum as in train_epoch: before
    epoch E the fit and fused_area_loss (and the exact-area metric) cover lanes 0 and 1, the heads all four."""
    from .optim import FusedOptimizer
    from .Loss_crit import fused_area_loss
    from .Networks import utils as nutils
    if not isinstance(optimizer, FusedOptimizer):
        raise TypeError("train_epoch_bev runs the update in the graph: it needs an optim.FusedOptimizer "
                        "(define_optim(..., fused=True)), got %s" % type(optimizer).__name__)
    check_bev_args(args)
    e2e, L, wf = bool(args.end_to_end), args.nclasses, args.weight_funct
    meters = DeviceMeters(("loss", "area", "exact"), next(model.parameters()).device)
    static = {}
    K = (curriculum_lanes(args, epoch) if e2e else None) or L     # --lane_curriculum, as in train_epoch

    def loss_fn(out):
        if e2e:
            loss, static["exact"] = fused_area_loss(out[:K], static["params"], wf, exact=True)
            if args.clas:
                loss = clas_loss(loss, out, static, criterion_line_class, criterion_horizon, args)
            return loss
        with torch.no_grad():
            static["area"], static["exact"] = fused_area_loss(out[:2], static["params"], wf, exact=True)
        return criterion_seg(out[6], static["gt"])

    def post(out, loss):
        ok = model.lsq_status.reshape(()).eq(0)
        n = static["input"].shape[0]
        if not e2e:
            meters.update("area", static["area"], ok, n)
        meters.update("loss", loss, ok, n)
        meters.update("exact", static["exact"], ok, n)
        return out

    def report(i, printing, saving, batch, out, bt):
        if printing:
            m = meters.read()
            print('Epoch: [{0}][{1}/{2}]\t'
                  'Time {3:.3f} ({4:.3f})\t'
                  'Loss {loss[0]:.8f} ({loss[1]:.8f})'.format(
                      epoch + 1, i + 1, len(loader), bt[0], bt[1], loss=m["loss"]))
        if saving:
            from .Dataloader.Load_Data_new import get_homography
            p = static["params"]
            nutils.save_weightmap('train', out[5], get_homography(args.resize), out[4], *out[:4], p[:, 0, :], p[:, 1, :],
                                  p[:, 2, :], p[:, 3, :], batch[4], static["gt"], 0, i, static["input"], args.no_ortho,
                                  args.resize, args.save_path)

    fields = lambda b: {"input": b[0], "gt": b[1], "params": b[2], "gt_line": b[4], "gt_horizon": b[5]}
    with _FitLanes(model, K if K < L else None):
        step = _train_replays(loader, model, optimizer, static, fields, {"input": torch.float32}, post, report,
                              args.print_freq, args.save_freq, loss_fn=loss_fn, end_to_end=e2e)
    if step is None:
        return 0, 0, 0
    m = meters.read()
    return m["loss"][1], m["area"][1], m["exact"][1]
