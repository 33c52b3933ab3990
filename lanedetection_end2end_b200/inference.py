"""Inference-side companions of the hot path (SURVEY.md 8f rank 1 / 4): what the reference's ``test.py`` does with the
curve coefficients after ``model(input, ...)``.

  Projections                BP/test.py:132-186  sample every fitted curve at the 56 TuSimple rows in BEV space and
                                                 project the samples back into the image with M^-1 -> x coordinates
  lanes_from_predictions     BP/test.py:66-86    gate lanes by the line-type / horizon heads, clip to the image
  write_tusimple_predictions BP/test.py:88-99    one JSON line per image in the TuSimple submission format

  lane_threshold             eval_lane.py:15-24,39  LaneEval's per-lane pixel threshold, bit-identical
  TuSimpleScorer             BP/test.py:66-99 + eval_lane.py:27-95  gating and LaneEval scoring on the GPU, one launch
                                                 (lf_tusimple_score, csrc/tusimple.cu) per batch
  test_model                 BP/test.py:23-129   the per-epoch test-set evaluation, one CUDA-graph replay per batch
  validate / validate_bev    BP/main.py:419-526, BEV/main.py:362-501  validation passes, one CUDA-graph replay per batch

``Projections.compute_coordinates`` keeps the reference's name, argument and result ([B, order+1, 1] float64 -> [B, 56]
float64, in 1280x720 pixels); on a CUDA tensor it is ONE launch of lf_backproj_loss (csrc/loss.cu, the kernel that
evaluates the training loss: same per-point code, x_cal output only) instead of two bmm's, a stack/permute and two
divisions; ``compute_all`` does all lanes of the batch in that one launch.
"""
import ctypes
import json
import os

import numpy as np
import torch

if __package__:
    from . import _capi
    from .Loss_crit import backprojection_loss, seg_confusion, seg_metrics_from_confusion
else:                                   # imported top-level next to the reference's main.py / test.py
    import _capi
    from Loss_crit import backprojection_loss, seg_confusion, seg_metrics_from_confusion

TUSIMPLE_SAMPLES = 56                   # h_samples 160..710 step 10: what Projections predicts
TUSIMPLE_LANES = 4                      # predicted lanes of the 4-lane --clas model
PIXEL_THRESH = 20                       # LaneEval.pixel_thresh (pt_thresh 0.85 lives in the kernel)


def resize_coordinates(array):
    """256x512 network coordinates -> 1280-wide TuSimple frames (BP/test.py:20-21)."""
    return array * 2.5


class Projections:
    """Back-projected lane x-coordinates at the TuSimple h_samples (BP/test.py:132-186)."""

    def __init__(self, options):
        if options.order > 3:
            raise NotImplementedError("Requested order {} for polynomial fit is not implemented".format(options.order))
        self._crit = backprojection_loss(options)      # owns Y56, y', M^-1 (the same constants, BP/Loss_crit.py:166-188)
        self.M, self.M_inv = self._crit.M, self._crit.M_inv

    def bind(self, model):
        """Project with ``model``'s learned warp (--learn_homography), read from its last forward."""
        self._crit.bind(model)
        return self

    def compute_all(self, betas):
        """betas: sequence of L tensors [B, order+1, 1] (Net.forward's beta0..3, None entries skipped) -> [B, L, 56] f64."""
        betas = [b for b in betas if b is not None]
        beta = torch.stack([b.reshape(b.shape[0], -1) for b in betas], 1).double().contiguous()       # [B, L, n]
        B, L, n = beta.shape
        if not beta.is_cuda:
            raise _capi.LanefitError("Projections runs on CUDA tensors (no CPU fallback by design)")
        dev = beta.device
        ones = torch.ones(B, L, 56, dtype=torch.float64, device=dev)
        zeros = torch.zeros(B, L, 56, dtype=torch.float64, device=dev)
        lane = torch.empty(L, dtype=torch.float64, device=dev)
        loss = torch.empty(1, dtype=torch.float64, device=dev)
        xcal = torch.empty(B, L, 56, dtype=torch.float64, device=dev)
        warp = self._crit.warp()
        if warp is not None:
            g = torch.empty(L + 1, 65, dtype=torch.float64, device=dev)
            _capi.call("lf_backproj_loss_dev", _capi.ptr(warp.yk.detach()), _capi.ptr(warp.Minv.detach()), _capi.ptr(beta),
                       _capi.ptr(zeros), _capi.ptr(ones), B, L, n, _capi.ptr(lane), _capi.ptr(loss),
                       _capi.ptr(torch.empty_like(beta)), _capi.ptr(xcal), _capi.ptr(g[:L]), _capi.ptr(g[L]),
                       _capi.ptr(self._crit._fused_ticket(dev)), _capi.stream_ptr())
            return resize_coordinates(xcal)
        host = self._crit._fused_host_constants()
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        _capi.call("lf_backproj_loss", host[0].ctypes.data, host[1].ctypes.data, host[2].ctypes.data, p(beta), p(zeros), p(ones),
                   B, L, n, p(lane), p(loss), None, p(xcal), p(self._crit._fused_ticket(dev)), _capi.stream_ptr())
        return resize_coordinates(xcal)

    def compute_coordinates(self, params):
        """params [B, order+1, 1] -> x coordinates [B, 56] in the 1280-wide frame (reference signature)."""
        return self.compute_all([params])[:, 0]


def lanes_from_predictions(x_cal, line_pred=None, horizon_pred=None):
    """x_cal [B, 4, 56] (Projections.compute_all) -> integer lane lists as the reference writes them (BP/test.py:66-86):
    lanes the line-type head switches off, samples above the predicted horizon and samples outside [0, 1279] become -2.
    line_pred [B, 4] in the head's order (rounded sigmoid); horizon_pred [B] in 720p rows (multiples of 10)."""
    lanes = x_cal.clone()
    if line_pred is not None:
        lp = line_pred[:, [1, 2, 0, 3]]
        lanes[(1 - lp[:, :, None]).bool().expand_as(lanes)] = -2
    if horizon_pred is not None:
        bounds = ((horizon_pred - 160) / 10)
        for k, bound in enumerate(bounds):
            lanes[k, :, :max(int(bound.item()), 0)] = -2
    lanes[lanes > 1279] = -2
    lanes[lanes < 0] = -2
    return np.int_(np.round(lanes.detach().cpu().numpy())).tolist()


def write_tusimple_predictions(json_file, gt_lines, lanes_pred, first_index, run_time=20):
    """Append one TuSimple submission line per image (BP/test.py:88-99; `run_time` is the reference's constant 20)."""
    for j, lanes in enumerate(lanes_pred):
        line = dict(gt_lines[first_index + j])
        line["lanes"] = lanes
        line["run_time"] = run_time
        json.dump(line, json_file)
        json_file.write("\n")


def lane_threshold(xs, h_samples):
    """LaneEval's pixel threshold of one ground-truth lane (eval_lane.py:15-24,39): 20 / cos(arctan(k)), k the slope of the
    least-squares line x = k y + c through the samples with x >= 0 (theta 0 below two of them).  sklearn's LinearRegression
    fits that line by centring y and x and calling scipy.linalg.lstsq; the same call here gives the same bits."""
    import scipy.linalg
    xs, ys = np.asarray(xs), np.asarray(h_samples)
    keep = xs >= 0
    theta = 0
    if int(keep.sum()) > 1:
        y = ys[keep].astype(np.float64)[:, None]
        x = xs[keep].astype(np.float64)
        y = y - np.average(y, axis=0)
        x = x - np.average(x)
        theta = np.arctan(scipy.linalg.lstsq(y, x, cond=1e-6)[0][0])
    return float(PIXEL_THRESH / np.cos(theta))


class TuSimpleScorer:
    """The TuSimple metric of a test pass on the GPU (BP/test.py:66-99 then LaneEval.bench_one_submit, eval_lane.py:59-95).

    Construction parses the ground truth (a test_label.json path or its parsed rows) once: every row must have 56
    h_samples (the rows Projections predicts; TuSimple's 48-sample 0313 clips are rejected, as LaneEval rejects them), lanes
    of len(h_samples) samples, at most 8 lanes and a unique raw_file; each lane's threshold is computed here
    (lane_threshold).  ``score`` is one lf_tusimple_score launch per batch: it gates and rounds the batch's lanes exactly as
    lanes_from_predictions does and scores them against rows pos .. pos + B - 1 exactly as LaneEval.bench does, then
    advances pos by B on the device, so it can be captured into a CUDA graph and replayed once per batch.  ``result``
    returns [accuracy, fp, fn] bit-identical to bench_one_submit on the file ``write_json`` writes."""

    def __init__(self, gt_rows_or_path, device="cuda"):
        if isinstance(gt_rows_or_path, (str, bytes, os.PathLike)):
            with open(gt_rows_or_path) as f:
                rows = [json.loads(line) for line in f.readlines()]
        else:
            rows = list(gt_rows_or_path)
        N, G, S = len(rows), _capi.TUSIMPLE_MAX_GT, TUSIMPLE_SAMPLES
        if N == 0:
            raise ValueError("the ground truth has no rows")
        gt_x = np.full((N, G, S), -2, np.int32)
        gt_n = np.zeros(N, np.int32)
        thresh = np.zeros((N, G), np.float64)
        seen = set()
        for i, row in enumerate(rows):
            name = row.get("raw_file")
            if name is None or "lanes" not in row or "h_samples" not in row:
                raise ValueError("ground-truth row %d lacks raw_file, lanes or h_samples" % i)
            if name in seen:
                raise ValueError("%s: duplicate raw_file in the ground truth" % name)
            seen.add(name)
            h, lanes = row["h_samples"], row["lanes"]
            if len(h) != S:
                raise ValueError("%s: %d h_samples; the predictions have %d (LaneEval raises 'Format of lanes error')"
                                 % (name, len(h), S))
            if len(lanes) > G:
                raise ValueError("%s: %d lanes, the table holds %d" % (name, len(lanes), G))
            for j, lane in enumerate(lanes):
                if len(lane) != len(h):
                    raise ValueError("%s: lane %d has %d samples for %d h_samples" % (name, j, len(lane), len(h)))
                arr = np.asarray(lane)
                if arr.dtype.kind not in "iu" or arr.min() < -2 ** 31 or arr.max() >= 2 ** 31:
                    raise ValueError("%s: lane %d holds values that are not int32 pixel columns" % (name, j))
                gt_x[i, j] = arr
                thresh[i, j] = lane_threshold(arr, h)
            gt_n[i] = len(lanes)
        dev = torch.device(device)
        self.rows, self.N = rows, N
        self.gt_x = torch.from_numpy(gt_x).to(dev)
        self.gt_lanes = torch.from_numpy(gt_n).to(dev)
        self.thresh = torch.from_numpy(thresh).to(dev)
        self.lanes = torch.full((N, TUSIMPLE_LANES, S), -2, dtype=torch.int32, device=dev)
        # per_image rows and pos share one buffer so that result() is one device-to-host copy
        self._out = torch.zeros(N * 3 + 1, dtype=torch.float64, device=dev)
        self.per_image = self._out[:N * 3].view(N, 3)
        self.pos = self._out[N * 3:].view(torch.int32)[:1]

    def score(self, x_cal, line_pred=None, horizon_pred=None):
        """x_cal [B, 4, 56] float64 (Projections.compute_all), line_pred [B, 4] float32 in the head's order (rounded
        sigmoid), horizon_pred [B] int32 (720p rows): one launch, no synchronisation."""
        B = x_cal.shape[0]
        if x_cal.dtype != torch.float64 or tuple(x_cal.shape[1:]) != (TUSIMPLE_LANES, TUSIMPLE_SAMPLES):
            raise ValueError("x_cal must be float64 [B, %d, %d], got %s %s" % (TUSIMPLE_LANES, TUSIMPLE_SAMPLES, x_cal.dtype,
                                                                               tuple(x_cal.shape)))
        if line_pred is not None and (line_pred.dtype != torch.float32 or tuple(line_pred.shape) != (B, TUSIMPLE_LANES)):
            raise ValueError("line_pred must be float32 [B, 4], got %s %s" % (line_pred.dtype, tuple(line_pred.shape)))
        if horizon_pred is not None and (horizon_pred.dtype != torch.int32 or tuple(horizon_pred.shape) != (B,)):
            raise ValueError("horizon_pred must be int32 [B], got %s %s" % (horizon_pred.dtype, tuple(horizon_pred.shape)))
        _capi.require_cuda(x_cal, line_pred, horizon_pred)
        c = lambda t: None if t is None else t.contiguous()
        x_cal, line_pred, horizon_pred = c(x_cal), c(line_pred), c(horizon_pred)
        p = _capi.ptr
        _capi.call("lf_tusimple_score", p(x_cal), p(line_pred), p(horizon_pred), B, TUSIMPLE_LANES, TUSIMPLE_SAMPLES,
                   p(self.gt_x), p(self.gt_lanes), p(self.thresh), self.N, _capi.TUSIMPLE_MAX_GT, p(self.pos), p(self.lanes),
                   p(self.per_image), _capi.stream_ptr())

    def reset(self):
        """Start a new pass at file row 0 (on the current stream)."""
        self.pos.zero_()

    def result(self):
        """[accuracy, fp, fn] of the pass as bench_one_submit returns them: the per-image rows summed in file order.  Raises
        unless every row was scored."""
        out = self._out.cpu().numpy()
        scored = min(int(out[self.N * 3:].view(np.int32)[0]), self.N)
        if scored != self.N:
            raise RuntimeError("scored %d of the %d ground-truth rows: LaneEval needs a prediction for every test image"
                               % (scored, self.N))
        accuracy, fp, fn = 0., 0., 0.
        for a, p, n in out[:self.N * 3].reshape(self.N, 3).tolist():
            accuracy += a
            fp += p
            fn += n
        return [accuracy / self.N, fp / self.N, fn / self.N]

    def predictions(self):
        """The gated integer lanes of every row (one copy), as lanes_from_predictions returns them."""
        return self.lanes.cpu().tolist()

    def write_json(self, json_file):
        write_tusimple_predictions(json_file, self.rows, self.predictions(), 0)


_SCORERS = {}           # (absolute path, device) -> (file stamp, TuSimpleScorer): one table build per ground-truth file


def _scorer_for(gt_file, device):
    st = os.stat(gt_file)
    key, stamp = (os.path.abspath(gt_file), str(device)), (st.st_mtime_ns, st.st_size)
    hit = _SCORERS.get(key)
    if hit is None or hit[0] != stamp:
        hit = _SCORERS[key] = (stamp, TuSimpleScorer(gt_file, device))
    return hit[1]


def test_model(loader, model, criterion, criterion_seg, criterion_line_class, criterion_horizon, args, epoch=0):
    """The reference's per-epoch test-set evaluation (BP/test.py:23-129), same signature and return value (the TuSimple
    accuracy).  Reads args.test_dir/test_label.json, writes args.save_path/test_set_predictions.json.

    Each batch is one CUDA-graph replay of the eval forward, the heads' post-processing (the reference's torch ops),
    Projections.compute_all and TuSimpleScorer.score; the host only copies the batch into the static input (a shorter last
    batch fills the leading slots and only its rows are scored).  Nothing synchronises until the end of the pass, where a
    singular least-squares system raises the RuntimeError the reference raises at its batch, the file is written and the
    accuracy line is printed.  Only the end-to-end 4-lane --clas model is scored, as in the reference; draw_testset (cv2
    drawing) is not supported."""
    if not (args.end_to_end and args.clas and args.nclasses == 4):
        raise ValueError("test_model scores the end-to-end 4-lane --clas model (end_to_end=%s, clas=%s, nclasses=%s)"
                         % (args.end_to_end, args.clas, args.nclasses))
    if args.draw_testset:
        raise NotImplementedError("draw_testset is not supported")
    if __package__:
        from .engine import GraphedInference
    else:
        from engine import GraphedInference
    dev = next(model.parameters()).device
    scorer = _scorer_for(os.path.join(args.test_dir, "test_label.json"), dev)
    params = Projections(args)
    if getattr(args, "learn_homography", False):
        params.bind(model)

    def post(out):
        horizon_pred = torch.sigmoid(out[7]).sum(dim=1)
        horizon_pred = (torch.round((resize_coordinates(horizon_pred) + 80) / 10) * 10).int()
        line_pred = torch.round(torch.sigmoid(out[6]))
        scorer.score(params.compute_all(out[:4]), line_pred, horizon_pred)

    deferred = model.defer_status_check
    graph, images, batches = None, 0, 0
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    try:
        with torch.no_grad():
            for batch in loader:
                n = batch.shape[0]
                if graph is None:
                    graph = GraphedInference(model, batch.to(dev, torch.float32), post=post)
                    scorer.reset()
                    model.lsq_status.zero_()
                    start.record()
                elif n > graph.x.shape[0]:
                    raise ValueError("batch of %d images after a first batch of %d" % (n, graph.x.shape[0]))
                graph.x[:n].copy_(batch, non_blocking=True)
                graph.graph.replay()
                images += n
                batches += 1
            end.record()
        if graph is None:
            raise ValueError("the test loader yielded no batch")
        graph.check()
    finally:
        model.defer_status_check = deferred
    if images != scorer.N:
        raise RuntimeError("We do not get the predictions of all the test tasks: %d images for %d ground-truth rows"
                           % (images, scorer.N))
    with open(os.path.join(args.save_path, "test_set_predictions.json"), "w") as f:
        scorer.write_json(f)
    acc_seg = scorer.result()
    print(acc_seg)
    print("===> Average ACC on TESTSET is {:.8} in {:.6}s for a batch".format(acc_seg[0], start.elapsed_time(end) / 1e3 / batches))
    return acc_seg[0]


def validate(loader, model, criterion, criterion_seg, criterion_line_class, criterion_horizon, args, epoch=0,
             seg_metrics=None):
    """The reference's validation pass (BP/main.py:419-526), same return value: (losses.avg, acc_hor_tot.avg,
    acc_line_tot.avg, rmse_metric_valid.avg).  ``args`` is main.py's global args, passed in.

    The loader yields the valid loader's 8-tuples (input, gt, lanes, idx, gt_line, gt_horizon, index, valid_points), on the
    device as Dataloader.Load_Data_new gives them (host tensors are copied in).  Each batch is one replay of a
    GraphedInference whose post= hook holds the per-lane criterion calls in main.py's order, with --clas the rounded-sigmoid
    accuracies (divided by resize * val_batch_size and nclasses * val_batch_size, also for a short batch), with --end_to_end
    False criterion_seg and the rmse metric, and the meter updates (engine.DeviceMeters) guarded by the LSQ status word: a
    batch with a singular system updates no meter, as main.py's `continue` does, and its line is printed at the end of the
    pass.  A batch shorter than the first (a loader that keeps its last batch) is replayed by a second graph of its size,
    so its losses are the ones main.py computes on it.  The host synchronises only at the print_freq lines, at
    save_weightmap('valid', ...) every 25 batches (called with the static outputs) and at the end.  The --clas BCE losses
    main.py adds after losses.update change nothing it returns and are not computed.

    A model built with --seg_proxy (``model.seg_proxy``) also scores its proxy segmentation branch in each replay, guarded
    like the meters: criterion_seg(output_seg, gt) into a device meter and Loss_crit.seg_confusion into the pass's
    [L+1, L+1] (target, prediction) count matrix.  At the end of the pass one more line is printed (proxy cross-entropy,
    pixel accuracy, per-class IoU and mIoU over the classes with a nonzero denominator) and a dict passed as
    ``seg_metrics`` receives "ce", "pixel_acc", "iou", "miou" and "confusion".  The returned tuple is unchanged."""
    if __package__:
        from .engine import GraphedInference, DeviceMeters, BatchStatus, lane_losses, _reporting
        from .Networks import utils as nutils
    else:
        from engine import GraphedInference, DeviceMeters, BatchStatus, lane_losses, _reporting
        from Networks import utils as nutils
    if args.clas and not args.end_to_end:
        raise ValueError("--clas needs --end_to_end True (the heads run on the end-to-end branch only)")
    e2e, L = bool(args.end_to_end), args.nclasses
    if not e2e and L != 4:
        raise ValueError("--end_to_end False needs 4 lanes: the reference's gt_line substitution does not broadcast the "
                         "loader's 4 line flags over %d lane maps" % L)
    if getattr(criterion, "learn_homography", False):
        criterion.bind(model)
    dev = next(model.parameters()).device
    proxy = bool(getattr(model, "seg_proxy", False))
    meters = DeviceMeters(("loss", "acc_hor", "acc_line", "rmse") + (("seg_proxy",) if proxy else ()), dev)
    status = BatchStatus(len(loader), dev)
    graphs = {}                     # rows -> (GraphedInference, static batch tensors)
    counts = torch.zeros((L + 1) ** 2, dtype=torch.int64, device=dev) if proxy else None

    def build(batch):
        st = {k: v.to(dev, non_blocking=True).clone() for k, v in batch.items()}
        st["input"], st["gt"] = st["input"].float(), st["gt"].long()
        n = st["input"].shape[0]

        def post(out):
            lanes, vp = st["lanes"], st["valid"]
            if e2e:
                loss, x_cal = lane_losses(criterion, out, lanes, vp, L)
            else:
                loss = criterion_seg(out[5], st["gt"])
                loss_metric, x_cal = lane_losses(criterion, out, lanes, vp, L)
            if proxy:
                ce = criterion_seg(out[8], st["gt"])
            if not torch.cuda.is_current_stream_capturing():
                return x_cal                 # warm-up passes: no meter or log entry
            ok = model.lsq_status.reshape(()).eq(0)
            if not e2e:
                meters.update("rmse", loss_metric, ok, n)
            meters.update("loss", loss, ok, n)
            if proxy:
                meters.update("seg_proxy", ce, ok, n)
                seg_confusion(out[8], st["gt"], counts, model.lsq_status)
            if args.clas:
                horizon_pred = torch.round(torch.nn.Sigmoid()(out[7]))
                acc = torch.eq(horizon_pred, st["gt_horizon"])
                acc_hor = torch.sum(acc).float() / (args.resize * args.val_batch_size)
                meters.update("acc_hor", acc_hor, ok)
                line_pred = torch.round(torch.nn.Sigmoid()(out[6]))
                acc = torch.eq(line_pred, st["gt_line"])
                acc_line = torch.sum(acc).float() / (args.nclasses * args.val_batch_size)
                meters.update("acc_line", acc_line, ok)
            status.record(model.lsq_status)
            model.lsq_status.zero_()
            return x_cal

        g = GraphedInference(model, st["input"], post=post, gt_line=None if e2e else st["gt_line"], end_to_end=e2e)
        st["input"] = g.x
        if not e2e:
            st["gt_line"] = g.gt_line        # the forward's substitution and the accuracies read one buffer
        model.lsq_status.zero_()
        return g, st

    deferred = model.defer_status_check
    first, labels = None, []
    try:
        with torch.no_grad():
            for i, (input, gt, lanes, idx, gt_line, gt_horizon, index, valid_points) in enumerate(loader):
                batch = {"input": input, "gt": gt.squeeze(1), "lanes": lanes, "gt_line": gt_line, "gt_horizon": gt_horizon,
                         "valid": valid_points}
                n = input.shape[0]
                status.check(i)
                if first is None:
                    first = n
                elif n > first:
                    raise ValueError("batch of %d images after a first batch of %d" % (n, first))
                if n in graphs:
                    g, st = graphs[n]
                    for k, v in batch.items():
                        st[k].copy_(v, non_blocking=True)
                else:
                    g, st = graphs[n] = build(batch)
                labels.append(idx)
                g.graph.replay()
                if not (_reporting(i, args.print_freq) or _reporting(i, 25)) or int(status.log[i]):
                    continue                     # a skipped batch reports nothing, as main.py's `continue`
                if _reporting(i, args.print_freq):
                    m = meters.read()
                    print('Test: [{0}/{1}]\t'
                          'Loss {loss[0]:.8f} ({loss[1]:.8f})\t'
                          'rmse {rmse[0]:.8f} ({rmse[1]:.8f})'.format(i + 1, len(loader), loss=m["loss"], rmse=m["rmse"]))
                if _reporting(i, 25):
                    lanes = st["lanes"]
                    nutils.save_weightmap('valid', g.out[4], *g.post_out, lanes[:, 0, :], lanes[:, 1, :], lanes[:, 2, :],
                                          lanes[:, 3, :], st["gt"], 0, i, st["input"], args.no_ortho, args.resize,
                                          args.save_path, args.nclasses, args.no_mapping)
    finally:
        model.defer_status_check = deferred
    m = meters.read()
    status.print_skipped(labels)
    if proxy:
        seg = seg_metrics_from_confusion(counts.view(L + 1, L + 1))
        seg["ce"] = m["seg_proxy"][1]
        print("===> Proxy segmentation on validation set: ENTROPY {:.8}  pixel acc {:.8}  IoU [{}]  mIoU {:.8}".format(
            seg["ce"], seg["pixel_acc"], ", ".join("{:.6}".format(v) for v in seg["iou"]), seg["miou"]))
        if seg_metrics is not None:
            seg_metrics.update(seg)
    if args.evaluate:
        crit_string = "TOT LOSS" if args.clas else ("MSE" if args.loss_policy == "backproject" and e2e else
                                                    "AREA**2" if args.loss_policy == "area" and e2e else "ENTROPY")
        print("===> Average {}-loss on validation set is {:.8}".format(crit_string, m["loss"][1]))
        if args.clas and len(loader) != 0:
            print("===> Average HORIZON ACC on val is {:.8}".format(m["acc_hor"][1]))
            print("===> Average LINE ACC on val is {:.8}".format(m["acc_hor"][1]))
    return m["loss"][1], m["acc_hor"][1], m["acc_line"][1], m["rmse"][1]


def validate_bev(loader, model, criterion, criterion_seg, criterion_line_class, criterion_horizon, M_inv, args, epoch=0):
    """The bird's-eye-view experiment's validation pass (Birds_Eye_View_Loss/main.py:362-501), same return value:
    (losses.avg, avg_area.avg, avg_trapezium_rule.avg, acc_hor_tot.avg, acc_line_tot.avg), the accuracies 0 (--clas is
    refused, engine.check_bev_args).

    The loader yields the BEV valid loader's 7-tuples (input, gt, params, idx, gt_line, gt_horizon, index), on the device
    as bev.Dataloader.Load_Data_new gives them.  Each batch is one replay of a GraphedInference whose post= hook holds
    Loss_crit.fused_area_loss (the lanes' area loss and the exact-area metric, one launch), with --end_to_end False
    criterion_seg and the 2-lane area, and the meter updates guarded by the LSQ status word: a batch with a singular system
    updates no meter, as main.py's `continue` does, and its line is printed at the end of the pass.  A batch shorter than
    the first is replayed by a second graph of its size.  The host synchronises only at the print_freq lines, at
    save_weightmap('valid', ...) every 25 batches and at the end."""
    if __package__:
        from .engine import GraphedInference, DeviceMeters, BatchStatus, _reporting, check_bev_args
        from .Loss_crit import fused_area_loss
        from .Networks import utils as nutils
    else:
        from engine import GraphedInference, DeviceMeters, BatchStatus, _reporting, check_bev_args
        from Loss_crit import fused_area_loss
        from Networks import utils as nutils
    check_bev_args(args)
    e2e, L, wf = bool(args.end_to_end), args.nclasses, args.weight_funct
    dev = next(model.parameters()).device
    meters = DeviceMeters(("loss", "area", "exact"), dev)
    status = BatchStatus(len(loader), dev)
    graphs = {}                     # rows -> (GraphedInference, static batch tensors)

    def build(batch):
        st = {k: v.to(dev, non_blocking=True).clone() for k, v in batch.items()}
        st["input"] = st["input"].float()
        n = st["input"].shape[0]

        def post(out):
            if e2e:
                loss, exact = fused_area_loss(out[:L], st["params"], wf, exact=True)
            else:
                loss = criterion_seg(out[6], st["gt"])
                area, exact = fused_area_loss(out[:2], st["params"], wf, exact=True)
            if not torch.cuda.is_current_stream_capturing():
                return None                  # warm-up passes: no meter or log entry
            ok = model.lsq_status.reshape(()).eq(0)
            if not e2e:
                meters.update("area", area, ok, n)
            meters.update("exact", exact, ok, n)
            meters.update("loss", loss, ok, n)
            status.record(model.lsq_status)
            model.lsq_status.zero_()
            return None

        g = GraphedInference(model, st["input"], post=post, end_to_end=e2e)
        st["input"] = g.x
        model.lsq_status.zero_()
        return g, st

    deferred = model.defer_status_check
    first, labels = None, []
    try:
        with torch.no_grad():
            for i, (input, gt, params, idx, gt_line, gt_horizon, index) in enumerate(loader):
                batch = {"input": input, "gt": gt, "params": params}
                n = input.shape[0]
                status.check(i)
                if first is None:
                    first = n
                elif n > first:
                    raise ValueError("batch of %d images after a first batch of %d" % (n, first))
                if n in graphs:
                    g, st = graphs[n]
                    for k, v in batch.items():
                        st[k].copy_(v, non_blocking=True)
                else:
                    g, st = graphs[n] = build(batch)
                labels.append(idx)
                g.graph.replay()
                if not (_reporting(i, args.print_freq) or _reporting(i, 25)) or int(status.log[i]):
                    continue                     # a skipped batch reports nothing, as main.py's `continue`
                if _reporting(i, args.print_freq):
                    m = meters.read()
                    print('Test: [{0}/{1}]\t'
                          'Loss {loss[0]:.8f} ({loss[1]:.8f})\t'
                          'Area {area[0]:.8f} ({area[1]:.8f})'.format(i + 1, len(loader), loss=m["loss"], area=m["area"]))
                if _reporting(i, 25):
                    out, p = g.out, st["params"]
                    nutils.save_weightmap('valid', out[5], M_inv, out[4], *out[:4], p[:, 0, :], p[:, 1, :], p[:, 2, :],
                                          p[:, 3, :], gt_line, st["gt"], 0, i, st["input"], args.no_ortho, args.resize,
                                          args.save_path)
    finally:
        model.defer_status_check = deferred
    m = meters.read()
    status.print_skipped(labels)
    if args.evaluate:
        crit_string = "AREA**2" if e2e else "ENTROPY"
        print("===> Average {}-loss on validation set is {:.8}".format(crit_string, m["loss"][1]))
        print("===> Average exact area on validation set is {:.8}".format(m["exact"][1]))
        if not e2e:
            print("===> Average area**2 on validation set is {:.8}".format(m["area"][1]))
    return m["loss"][1], m["area"][1], m["exact"][1], 0, 0
