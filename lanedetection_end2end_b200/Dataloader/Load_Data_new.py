"""The reference's TuSimple loader (BP/Dataloader/Load_Data_new.py) on the GPU, with the same public names and signatures:

    from Dataloader.Load_Data_new import get_loader, get_testloader, load_valid_set_file_all
    train_loader, valid_loader, valid_idx = get_loader(num_train, json_file, lanes_file, image_dir, gt_dir, flip_on,
                                                       batch_size, val_batch_size, shuffle, num_workers, end_to_end,
                                                       resize, nclasses)
    for image, gt, lanes, idx, line_lst, horizon, valid_points in train_loader:   # device tensors; idx on the CPU
        ...

A batch is the reference's collated tuple, element by element: image float32 [N,3,R,2R], gt int64 [N,1,R,2R], lanes
float64 [N,4,56], idx int64 (CPU), line_lst float32 [N,4], horizon float32 [N,R], index int64 (CPU; validation samples
only), valid_points float64 [N,4,56], all bit-identical to the reference's.  The test loader yields image batches
float32 [N,3,R,2R] and keeps the short last batch.

How a batch is made:
  * Order: a torch DataLoader over the sample indices, with the reference's sampler, batch_size and drop_last, so the
    torch RNG is consumed as the reference's DataLoader consumes it (the iterator's base seed, then SubsetRandomSampler's
    randperm).  get_loader's np.random.seed(num_train) shuffle and split are the reference's.
  * Flips: one np.random.uniform(0.0, 1.0) per sample, in sample order, in the main process, when the batch is requested,
    drawn even when flip_on is off or the sample is a validation sample -- the reference's draws with num_workers=0.
    With num_workers > 0 the reference draws from per-worker numpy seeds; that sequence is not reproduced.  Here
    num_workers is the number of host threads that read files.
  * Decoding (jpeg.JpegDecoder, png.PngDecoder) and crop + resize (lf_loader_stage) run on a side stream one batch ahead,
    into slots of uint8 buffers of resized, unflipped samples.  The flip comes at assembly (lf_loader_assemble, on the
    consumer's current stream after it waits for the staging), so prefetching changes no draw.
  * Cache: each dataset owns one.  When all its resized samples fit `cache_bytes` (default 4 GiB, or the environment
    variable LANEFIT_LOADER_CACHE_BYTES; 0 disables) every sample has its own slot, and once the epoch that filled a slot
    has ended with clean decoder checks, the slot is served without file I/O, parsing or decoding.  Otherwise two staging
    buffers alternate.  The decoders' status words are read at the end of every epoch that decoded (the only host
    synchronisation): a corrupt file raises ValueError then, and the slots filled in that epoch are decoded again next
    epoch.
  * Label elements come from per-sample tables built once on the host with the reference's own float64 expressions, for
    both flip states, gathered by the assembly launch.

Reference behaviour kept: the string sort of the file names and label row int(name) - 1, the -2 left padding of
48-sample rows and the misaligned horizon zip, the /2.5 and -32 rescale that ignores `resize`, valid_points neither
flipped nor permuted, line types through mirror_list, the 3 / 4 quirk of the flipped gt, nclasses < 3 zeroing classes 3
and 4 before the flip, and the 3626-file assert.  Differences: len() works; files the decoders do not support (and mixed
frame sizes, or a label map whose size differs from its frame's) raise ValueError naming the file -- there is no Pillow
fallback.  Keyword-only extras: device, cache_bytes, expected_count (None: any number of files), line_file."""
import json
import os
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset
from torch.utils.data.sampler import Sampler

from lanedetection_end2end_b200 import _capi, jpeg, png
from lanedetection_end2end_b200.input_pipeline import FramePreprocessor, LabelPreprocessor

CACHE_ENV = "LANEFIT_LOADER_CACHE_BYTES"
DEFAULT_CACHE_BYTES = 4 << 30
CROP_ROWS = 640
NUM_POINTS = _capi.LOADER_POINTS
NUM_LANES = _capi.LOADER_LANES

BatchPlan = namedtuple("BatchPlan", "positions rows draws flips index")
BatchPlan.__doc__ = """One batch as the iteration makes it: dataset positions, label rows (the reference's `idx`), the
np.random.uniform draw of each sample, the flip applied (draw > 0.5, flip_on, not a validation sample), and the validation
`index` of each sample (None for a training batch)."""


def default_cache_bytes():
    v = os.environ.get(CACHE_ENV)
    return DEFAULT_CACHE_BYTES if v is None or v == "" else int(v)


# ---------------------------------------------------------------------------------------------------------------------
# host label tables (Load_Data_new.py:133-158,176-192 of the reference, per label row, for both flip states)

def _line_types(line_lst):
    line = np.array(line_lst[3:7])
    return torch.from_numpy(np.array(line + 1)).clamp(0, 1).float().numpy()


def label_row(lanes_lst, h_samples, line_lst, resize):
    """The label elements of one sample: (lanes unflipped, lanes flipped) float64 [4,56], valid_points float64 [4,56],
    the number of leading ones of horizon, (line_lst unflipped, flipped) float32 [4].  The reference's expressions."""
    lanes = np.array(lanes_lst)
    to_add = np.full((4, 56 - lanes.shape[1]), -2)
    lanes = np.hstack((to_add, lanes))
    valid_points = np.int32(lanes > 0)
    valid_points[:, :8] = 0
    lanes = lanes / 2.5
    track = lanes < 0
    h_samples = np.array(h_samples) / 2.5 - 32
    lanes[track] = -2
    horizon_lanes = []
    for lane in lanes:
        horizon_lanes.append(min([y_cord for (x_cord, y_cord) in zip(lane, h_samples) if x_cord != -2] or [resize]))
    y_val = min(horizon_lanes)
    nhorizon = len(range(resize)[0:int(np.floor(y_val))])       # torch.zeros(resize)[0:k] = 1, slice semantics
    flipped = (2 * resize - 1) - lanes
    flipped[track] = -2
    flipped = flipped[[1, 0, 3, 2]]
    return ((lanes.astype(np.float64), flipped.astype(np.float64)), valid_points.astype(np.float64), nhorizon,
            (_line_types(line_lst), _line_types(mirror_list(line_lst))))


def label_tables(ordered_lanes, line_file, rows, resize):
    """Tables over the dataset positions whose label rows are `rows`: lanes float64 [2,P,4,56] (unflipped, flipped),
    valid float64 [P,4,56], horizon int32 [P] (leading ones of the horizon vector), line float32 [2,P,4]."""
    P = len(rows)
    lanes = np.empty((2, P, NUM_LANES, NUM_POINTS), np.float64)
    valid = np.empty((P, NUM_LANES, NUM_POINTS), np.float64)
    horizon = np.empty(P, np.int32)
    line = np.empty((2, P, NUM_LANES), np.float32)
    for p, r in enumerate(rows):
        (l0, l1), v, h, (c0, c1) = label_row(ordered_lanes[r]["lanes"], ordered_lanes[r]["h_samples"], line_file[r]["lines"],
                                             resize)
        lanes[0, p], lanes[1, p], valid[p], horizon[p], line[0, p], line[1, p] = l0, l1, v, h, c0, c1
    return {"lanes": lanes, "valid": valid, "horizon": horizon, "line": line}


def horizon_vectors(nhorizon, resize):
    """float32 [P, resize] horizon vectors from the table's counts."""
    return (np.arange(resize)[None, :] < np.asarray(nhorizon)[:, None]).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# device store: decoders, slots, staging and assembly

def _read(path):
    with open(path, "rb") as f:
        return f.read()


class _SampleStore:
    """Slot-addressed uint8 buffers of resized, unflipped samples on one device, and the decoders that fill them.
    Slot state: 0 empty, 1 filled in the current epoch (not served until the decoders' check at its end), 2 served.

    label_rows (the bird's-eye-view loader): after staging, lf_loader_label_rows records the first labelled row of each new
    map in `first_row` (device int32, per dataset position).  The end-of-epoch check copies it to the host and raises
    ValueError for every map served in the epoch that has no labelled pixel."""

    def __init__(self, frame_paths, map_paths, resize, device, cache_bytes, label_rows=False):
        self.frame_paths, self.map_paths = list(frame_paths), None if map_paths is None else list(map_paths)
        self.P, self.R = len(self.frame_paths), int(resize)
        self.Ho, self.Wo = self.R, 2 * self.R
        per = self.Ho * self.Wo * (3 + (0 if self.map_paths is None else 1))
        budget = default_cache_bytes() if cache_bytes is None else int(cache_bytes)
        self.cached = 0 < budget and self.P * per <= budget
        self.device = device
        self.state = np.zeros(self.P, np.int8)
        self.label_rows = label_rows
        self.first_row_host = np.full(self.P, -2, np.int32) if label_rows else None   # -2: not recorded yet
        self._served = np.zeros(self.P, bool) if label_rows else None
        self.workers = 0
        self._pool = None
        self._dev = None

    # lazily, on the first batch: no device work before the first iteration
    def _setup(self):
        if self._dev is not None:
            return
        dev = torch.device(self.device if self.device is not None else "cuda")
        if dev.type != "cuda":
            raise _capi.LanefitError("the loader runs on CUDA only; got device %s" % dev)
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self._dev = dev
        self.jdec = jpeg.JpegDecoder(dev)
        self.pdec = None if self.map_paths is None else png.PngDecoder(dev)
        self.side = torch.cuda.Stream(dev)
        self.frame_hw, self.fpre, self.lpre = None, None, None
        self.frames = self.maps = None
        self.capacity = 0
        if self.cached:
            self._alloc(self.P)
        self._ring = 0
        self._ring_read = [None, None]   # per staging buffer: event of the last assembly that read it
        self._assembled = {}             # consumer stream -> event of its last assembly (cache mode)
        self._decoded = False
        self.first_row = None
        if self.label_rows:
            with torch.cuda.stream(self.side):     # ordered before the side stream's lf_loader_label_rows
                self.first_row = torch.full((self.P,), -2, dtype=torch.int32, device=dev)

    def _alloc(self, S):
        self.frames = torch.empty(S, self.Ho, self.Wo, 3, dtype=torch.uint8, device=self._dev)
        self.maps = None if self.map_paths is None else torch.empty(S, self.Ho, self.Wo, dtype=torch.uint8, device=self._dev)
        self.capacity = S

    def _decode(self, decoder, parse, datas, paths):
        try:
            return decoder(datas)
        except ValueError as e:
            sizes = []
            for p, d in zip(paths, datas):
                try:
                    h = parse(d)
                except ValueError as e1:
                    raise ValueError("%s: %s" % (p, e1)) from None
                sizes.append((h.width, h.height))
                if sizes[-1] != sizes[0]:
                    raise ValueError("%s: %dx%d, but %s is %dx%d" % (p, sizes[-1][0], sizes[-1][1], paths[0], sizes[0][0],
                                                                   sizes[0][1])) from None
            raise ValueError("%s: %s" % (", ".join(paths), e)) from None

    def _check_size(self, hw, paths, what):
        if self.frame_hw is None:
            if hw[0] < CROP_ROWS:
                raise ValueError("%s: %s of %dx%d; the loader crops the bottom %d rows" % (paths[0], what, hw[1], hw[0], CROP_ROWS))
            self.frame_hw = hw
            self.fpre = FramePreprocessor(self.R, frame_hw=hw, crop_rows=CROP_ROWS, device=self._dev)
            self.lpre = LabelPreprocessor(self.R, 4, frame_hw=hw, crop_rows=CROP_ROWS, device=self._dev)
        elif hw != self.frame_hw:
            raise ValueError("%s: %s of %dx%d, the dataset's frames are %dx%d" % (paths[0], what, hw[1], hw[0], self.frame_hw[1],
                                                                                  self.frame_hw[0]))

    def stage(self, positions):
        """Decode and stage the samples of `positions` that the cache does not serve, on the side stream.  Returns
        (slot of each position, event the assembly waits for or None)."""
        self._setup()
        positions = list(positions)
        if self._served is not None:
            self._served[positions] = True
        if self.cached:
            slots = positions
            need = [k for k, p in enumerate(positions) if self.state[p] != 2]
        else:
            B = len(positions)
            if self.capacity < 2 * B:
                self._alloc(2 * B)
                self._ring_read = [None, None]
            r, self._ring = self._ring, self._ring ^ 1
            slots = [r * (self.capacity // 2) + k for k in range(B)]
            need = list(range(B))
        if not need:
            return slots, None
        fpaths = [self.frame_paths[positions[k]] for k in need]
        mpaths = None if self.map_paths is None else [self.map_paths[positions[k]] for k in need]
        allp = fpaths + (mpaths or [])
        datas = list(self._pool.map(_read, allp)) if self._pool is not None else [_read(p) for p in allp]
        fdat, mdat = datas[:len(fpaths)], datas[len(fpaths):]
        side = self.side
        with torch.cuda.stream(side):
            if self.cached:
                for ev in self._assembled.values():
                    side.wait_event(ev)
            elif self._ring_read[r] is not None:
                side.wait_event(self._ring_read[r])
            frames = self._decode(self.jdec, jpeg.parse, fdat, fpaths)
            self._decoded = True
            self._check_size(tuple(frames.shape[1:3]), fpaths, "frame")
            maps = None
            if mpaths is not None:
                maps = self._decode(self.pdec, png.parse, mdat, mpaths)
                if tuple(maps.shape[1:]) != self.frame_hw:
                    raise ValueError("%s: label map of %dx%d for a frame of %dx%d" % (mpaths[0], maps.shape[2], maps.shape[1],
                                                                                     self.frame_hw[1], self.frame_hw[0]))
            sl = torch.tensor([slots[k] for k in need], dtype=torch.int32).pin_memory().to(self._dev, non_blocking=True)
            H, W = self.frame_hw
            xb, xk, yb, yk = self.fpre.tables
            p = _capi.ptr
            _capi.call("lf_loader_stage", p(frames), p(maps), len(need), H, W, H - CROP_ROWS, CROP_ROWS, p(xb), p(xk), self.fpre.kx,
                       p(yb), p(yk), self.fpre.ky, p(self.lpre.xs), p(self.lpre.ys), self.Ho, self.Wo, p(sl), p(self.frames),
                       p(self.maps), _capi.stream_ptr(), nbytes=frames.numel() + (0 if maps is None else maps.numel())
                       + len(need) * self.Ho * self.Wo * 4)
            if self.first_row is not None:
                # a position staged again (ring mode, across an epoch boundary) rewrites the same value
                pos = torch.tensor([positions[k] for k in need], dtype=torch.int32).pin_memory().to(self._dev, non_blocking=True)
                _capi.call("lf_loader_label_rows", p(self.maps), len(need), self.Ho, self.Wo, p(sl), p(pos), p(self.first_row),
                           _capi.stream_ptr(), nbytes=len(need) * self.Ho * self.Wo)
            ev = torch.cuda.Event()
            ev.record(side)
        if self.cached:
            self.state[[positions[k] for k in need]] = 1
        return slots, ev

    def assembly_begin(self, slots, rows, flips, staged):
        """(current stream, device int32 [N][3] (slot, table row, flip)) for an assembly launch that reads the slots, after
        the current stream waits for `staged`.  The launch is followed by assembly_end."""
        stream = torch.cuda.current_stream(self._dev)
        if staged is not None:
            stream.wait_event(staged)
        sample = torch.from_numpy(np.stack([np.asarray(slots), np.asarray(rows), np.asarray(flips)], 1).astype(np.int32))
        return stream, sample.pin_memory().to(self._dev, non_blocking=True)

    def assembly_end(self, stream, slots):
        """Record that `stream` read the slots, so staging does not overwrite them before it has."""
        ev = torch.cuda.Event()
        ev.record(stream)
        if self.cached:
            self._assembled[stream] = ev
        else:
            self._ring_read[0 if slots[0] < self.capacity // 2 else 1] = ev
            for b in (self.frames, self.maps):
                if b is not None:
                    b.record_stream(stream)

    def assemble(self, slots, rows, flips, staged, nclasses, tables, image_only):
        """The batch's device elements on the current stream, from the slots (after `staged`)."""
        stream, sample = self.assembly_begin(slots, rows, flips, staged)
        N = len(slots)
        dev, R = self._dev, self.R
        image = torch.empty(N, 3, R, 2 * R, dtype=torch.float32, device=dev)
        out = [image]
        if image_only:
            gt = lanes = valid = horizon = line = None
            nrows = 0
        else:
            gt = torch.empty(N, 1, R, 2 * R, dtype=torch.int64, device=dev)
            lanes = torch.empty(N, NUM_LANES, NUM_POINTS, dtype=torch.float64, device=dev)
            valid = torch.empty(N, NUM_LANES, NUM_POINTS, dtype=torch.float64, device=dev)
            horizon = torch.empty(N, R, dtype=torch.float32, device=dev)
            line = torch.empty(N, NUM_LANES, dtype=torch.float32, device=dev)
            out += [gt, lanes, valid, horizon, line]
            nrows = tables["horizon"].shape[0]
        p = _capi.ptr
        t = tables or {}
        _capi.call("lf_loader_assemble", p(self.frames), p(self.maps), N, R, 2 * R, nclasses, p(sample), nrows, p(t.get("lanes")),
                   p(t.get("valid")), p(t.get("horizon")), p(t.get("line")), p(image), p(gt), p(lanes), p(valid), p(horizon),
                   p(line), _capi.stream_ptr(), nbytes=sum(o.numel() * o.element_size() for o in out) + N * R * 2 * R * 4)
        self.assembly_end(stream, slots)
        return out

    def finish_epoch(self):
        """End of an epoch: read the decoders' status words if anything was decoded since the last read; the slots filled
        since then are served from now on, or, after a corrupt file, emptied (and ValueError raised)."""
        if self._dev is None:
            return
        served = None
        if self._served is not None:
            served, self._served = self._served, np.zeros(self.P, bool)
        if self._decoded:
            self._check_decoders()
            if self.first_row is not None:
                with torch.cuda.stream(self.side):
                    self.first_row_host = self.first_row.cpu().numpy()
        if served is not None:
            bad = np.nonzero(served & (self.first_row_host == -1))[0]
            if len(bad):
                raise ValueError("%s: no labelled pixel (a value other than 0, 3 and 4) in the resized label map, so the "
                                 "horizon is undefined" % ", ".join(self.map_paths[i] for i in bad))

    def _check_decoders(self):
        self._decoded = False
        errors = []
        for d in (self.jdec, self.pdec):
            if d is not None:
                try:
                    d.check()
                except ValueError as e:
                    errors.append(str(e))
        pending = self.state == 1
        if errors:
            self.state[pending] = 0
            raise ValueError("; ".join(errors) + " (a file decoded in this epoch; its samples are decoded again next epoch)")
        self.state[pending] = 2

    def set_workers(self, n):
        n = int(n or 0)
        if n > self.workers:
            self.workers = n
            self._pool = ThreadPoolExecutor(max_workers=n)


# ---------------------------------------------------------------------------------------------------------------------
# datasets and loaders

class _Indices(Dataset):
    """The sample positions: the torch DataLoader over it makes the reference's order."""

    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return i


def _collate_positions(batch):
    return list(batch)


class LaneLoader:
    """Iterable over the collated device batches of a LaneDataset or LaneTestSet, in the order of a torch DataLoader with
    the same sampler / shuffle, batch_size and drop_last."""

    def __init__(self, dataset, batch_size=1, sampler=None, shuffle=False, num_workers=0, drop_last=False):
        self.dataset, self.batch_size, self.sampler, self.drop_last = dataset, batch_size, sampler, drop_last
        self.num_workers = num_workers
        self._order = DataLoader(_Indices(len(dataset)), batch_size=batch_size, sampler=sampler, shuffle=shuffle, num_workers=0,
                                 drop_last=drop_last, collate_fn=_collate_positions)
        dataset._store.set_workers(num_workers)

    def __len__(self):
        return len(self._order)

    def plans(self):
        """One epoch of BatchPlans, consuming the torch and numpy RNGs exactly as iterating the loader does, without a GPU."""
        for positions in self._order:
            yield self.dataset._plan(positions)

    def __iter__(self):
        return _LoaderIter(self)


class _LoaderIter:
    def __init__(self, loader):
        self.ds = loader.dataset
        self.order = iter(loader._order)          # the base seed is drawn here, as by the reference's iter(loader)
        self.ahead = None                         # (positions, staging) of the next batch
        self.done = False

    def __iter__(self):
        return self

    def __next__(self):
        if self.done:
            raise StopIteration
        if self.ahead is None:
            positions = next(self.order, None)
            if positions is None:
                return self._end()
            self.ahead = (positions, self.ds._store.stage(positions))
        positions, (slots, staged) = self.ahead
        self.ahead = None
        plan = self.ds._plan(positions)           # the flip draws, when the batch is requested
        batch = self.ds._assemble(plan, slots, staged)
        nxt = next(self.order, None)
        if nxt is not None:
            self.ahead = (nxt, self.ds._store.stage(nxt))
        return batch

    def _end(self):
        self.done = True
        self.ds._store.finish_epoch()
        raise StopIteration


class LaneDataset(Dataset):
    """Dataset with labeled lanes (the reference's LaneDataset).  Indexing returns one sample as the reference's
    __getitem__ does (device tensors, idx and index as ints), drawing its flip; it reads the decoders' status at once."""

    def __init__(self, end_to_end, valid_idx, json_file, lanes_file, image_dir, gt_dir, flip_on, resize, nclasses, *,
                 device=None, cache_bytes=None, expected_count=3626, line_file="Labels/label_new.json"):
        self.image_dir = image_dir
        self.gt_dir = gt_dir
        self.flip_on = flip_on
        self.resize = resize
        with open(json_file) as f:
            self.params = [json.loads(line) for line in f.readlines()]
        with open(lanes_file) as f:
            self.ordered_lanes = [json.loads(line) for line in f.readlines()]
        with open(line_file) as f:
            self.line_file = [json.loads(line) for line in f.readlines()]
        self.end_to_end = end_to_end
        self.rgb_lst = sorted(os.listdir(image_dir))
        self.gt_lst = sorted(os.listdir(gt_dir))
        self.num_imgs = len(self.rgb_lst)
        if expected_count is not None:
            assert len(self.rgb_lst) == len(self.gt_lst) == expected_count
        elif len(self.rgb_lst) != len(self.gt_lst):
            raise ValueError("%d images in %s but %d label maps in %s" % (len(self.rgb_lst), image_dir, len(self.gt_lst), gt_dir))
        for a, b in zip(self.rgb_lst, self.gt_lst):
            assert a.split(".")[0] == b.split(".")[0], (a, b)
        target_idx = [int(i.split(".")[0]) for i in self.rgb_lst]
        self.valid_idx = [target_idx[i] - 1 for i in valid_idx]
        self._valid_set = set(self.valid_idx)
        self.rows = [t - 1 for t in target_idx]
        self.num_points = 56
        self.nclasses = nclasses
        print("Flipping images randomly:", self.flip_on)
        print("End to end lane detection:", self.end_to_end)
        self.tables = label_tables(self.ordered_lanes, self.line_file, self.rows, int(resize))
        self._dev_tables = None
        self._store = _SampleStore([os.path.join(image_dir, n) for n in self.rgb_lst], [os.path.join(gt_dir, n) for n in self.gt_lst],
                                   resize, device, cache_bytes)

    def __len__(self):
        return self.num_imgs

    def _plan(self, positions):
        positions = list(positions)
        rows = [self.rows[p] for p in positions]
        draws, flips, index = [], [], []
        for r in rows:
            u = np.random.uniform(0.0, 1.0)
            draws.append(u)
            valid = r in self._valid_set
            flips.append(bool(not valid and (u > 0.5 and self.flip_on)))
            index.append(self.valid_idx.index(r) if valid else None)
        if any(i is None for i in index):
            if any(i is not None for i in index):
                raise ValueError("a batch mixes training and validation samples; the reference cannot collate it")
            index = None
        return BatchPlan(positions, rows, draws, flips, index)

    def _assemble(self, plan, slots, staged):
        st = self._store
        if self._dev_tables is None:
            st._setup()
            self._dev_tables = {k: torch.from_numpy(np.ascontiguousarray(v)).to(st._dev) for k, v in self.tables.items()}
        image, gt, lanes, valid, horizon, line = st.assemble(slots, plan.positions, [int(f) for f in plan.flips], staged,
                                                              self.nclasses, self._dev_tables, False)
        idx = torch.tensor(plan.rows, dtype=torch.int64)
        if plan.index is not None:
            return image, gt, lanes, idx, line, horizon, torch.tensor(plan.index, dtype=torch.int64), valid
        return image, gt, lanes, idx, line, horizon, valid

    def __getitem__(self, idx):
        slots, staged = self._store.stage([idx])
        batch = self._assemble(self._plan([idx]), slots, staged)
        self._store.finish_epoch()
        return tuple(int(t[0]) if t.device.type == "cpu" else t[0] for t in batch)


class LaneTestSet(Dataset):
    """Dataset used as testset (the reference's LaneTestSet): frames only, yielded as float32 [3,R,2R] device images."""

    def __init__(self, gt_file, resize, path, *, device=None, cache_bytes=None):
        with open(gt_file, "r") as f:
            self.img_info = [json.loads(line) for line in f]
        print("size test loader: ", len(self.img_info))
        self.path = path
        self.resize = resize
        self._store = _SampleStore([os.path.join(path, r["raw_file"]) for r in self.img_info], None, resize, device, cache_bytes)

    def __len__(self):
        return len(self.img_info)

    def _plan(self, positions):
        positions = list(positions)
        return BatchPlan(positions, positions, [], [False] * len(positions), None)

    def _assemble(self, plan, slots, staged):
        return self._store.assemble(slots, plan.positions, plan.flips, staged, 0, None, True)[0]

    def __getitem__(self, idx):
        slots, staged = self._store.stage([idx])
        image = self._assemble(self._plan([idx]), slots, staged)
        self._store.finish_epoch()
        return image[0]


def get_testloader(path, batch_size, num_workers, resize=256, *, device=None, cache_bytes=None):
    json_file = os.path.join(path, "test_label.json")
    transformed_dataset = LaneTestSet(gt_file=json_file, path=path, resize=resize, device=device, cache_bytes=cache_bytes)
    return LaneLoader(transformed_dataset, batch_size=batch_size, shuffle=False, num_workers=num_workers, drop_last=False)


def mirror_list(lst):
    """Mirror lists of lane and line classification ground truth in order to make flipping possible"""
    middle = len(lst) // 2
    first = list(reversed(lst[:middle]))
    second = list(reversed(lst[middle:]))
    return second + first


def homogenous_transformation(Matrix, x, y):
    """Transform the points (x, y) by the 3x3 projective matrix `Matrix`; returns (x', y')."""
    ones = np.ones((1, len(y)))
    coordinates = np.vstack((x, y, ones))
    trans = np.matmul(Matrix, coordinates)
    return trans[0, :] / trans[2, :], trans[1, :] / trans[2, :]


def get_homography(resize=320):
    """The inverse of the loader's bird's-eye-view homography at `resize` (the reference returns M_inv only)."""
    import cv2
    y_start = 0.3 * (resize - 1)
    y_stop = resize - 1
    src = np.float32([[0.45 * (2 * resize - 1), y_start], [0.55 * (2 * resize - 1), y_start], [0.1 * (2 * resize - 1), y_stop],
                      [0.9 * (2 * resize - 1), y_stop]])
    dst = np.float32([[0.45 * (2 * resize - 1), y_start], [0.55 * (2 * resize - 1), y_start], [0.45 * (2 * resize - 1), y_stop],
                      [0.55 * (2 * resize - 1), y_stop]])
    return cv2.getPerspectiveTransform(dst, src)


class SequentialIndicesSampler(Sampler):
    def __init__(self, indices):
        self.indices = indices

    def __iter__(self):
        return iter(self.indices)

    def __len__(self):
        return len(self.indices)


def get_loader(num_train, json_file, lanes_file, image_dir, gt_dir, flip_on, batch_size, val_batch_size, shuffle, num_workers,
               end_to_end, resize, nclasses, split_percentage=0.2, *, device=None, cache_bytes=None, expected_count=3626,
               line_file="Labels/label_new.json"):
    """Split the dataset into training and validation samples and make their loaders (one dataset, one cache)."""
    indices = list(range(num_train))
    split = int(np.floor(split_percentage * num_train))
    if shuffle is True:
        np.random.seed(num_train)
        np.random.shuffle(indices)
    train_idx, valid_idx = indices[split:], indices[:split]
    print("size train loader is", len(train_idx))
    print("size valid loader is", len(valid_idx))
    train_sampler = torch.utils.data.sampler.SubsetRandomSampler(train_idx)
    valid_sampler = SequentialIndicesSampler(valid_idx)
    transformed_dataset = LaneDataset(end_to_end=end_to_end, valid_idx=valid_idx, json_file=json_file, lanes_file=lanes_file,
                                      image_dir=image_dir, gt_dir=gt_dir, flip_on=flip_on, resize=resize, nclasses=nclasses,
                                      device=device, cache_bytes=cache_bytes, expected_count=expected_count, line_file=line_file)
    train_loader = LaneLoader(transformed_dataset, batch_size=batch_size, sampler=train_sampler, num_workers=num_workers,
                              drop_last=True)
    valid_loader = LaneLoader(transformed_dataset, batch_size=val_batch_size, sampler=valid_sampler, num_workers=num_workers,
                              drop_last=True)
    return train_loader, valid_loader, valid_idx


def _write_rows(target_file, labels_file, ids):
    with open(target_file, "w") as jsonFile:
        for image_id in ids:
            json.dump(labels_file[image_id], jsonFile)
            jsonFile.write("\n")


def _json_lines(path):
    with open(path) as f:
        return [json.loads(line) for line in f.readlines()]


def load_valid_set_file(valid_idx):
    """validation_set.json from the three TuSimple label files, indexed across them."""
    labels_file1 = _json_lines("Labels/label_data_0313.json")
    labels_file2 = _json_lines("Labels/label_data_0531.json")
    labels_file3 = _json_lines("Labels/label_data_0601.json")
    len_file1, len_file2 = len(labels_file1), len(labels_file2)
    rows = []
    for image_id in valid_idx:
        if image_id < len_file1:
            rows.append(labels_file1[image_id])
        elif image_id < len_file1 + len_file2:
            rows.append(labels_file2[image_id - len_file1])
        else:
            rows.append(labels_file3[image_id - len_file1 - len_file2])
    _write_rows("validation_set.json", rows, range(len(rows)))


def load_valid_set_file_all(valid_idx, target_file, image_dir):
    """`target_file` = the rows of Labels/label_data_all.json of the validation samples, mapped through the string-sorted
    file names of `image_dir` (row int(name) - 1)."""
    labels_file = _json_lines("Labels/label_data_all.json")
    content = sorted(os.listdir(image_dir))
    target_idx = [int(i.split(".")[0]) for i in content]
    _write_rows(target_file, labels_file, [target_idx[i] - 1 for i in valid_idx])


def load_0313_valid_set_file(valid_idx, nclasses):
    """validation_set.json from Labels/label_data_0313.json, keeping the first `nclasses` lanes of each row."""
    labels_file1 = _json_lines("Labels/label_data_0313.json")
    rows = []
    for image_id in valid_idx:
        labels = labels_file1[image_id]
        labels["lanes"] = labels["lanes"][0:nclasses]
        rows.append(labels)
    _write_rows("validation_set.json", rows, range(len(rows)))
