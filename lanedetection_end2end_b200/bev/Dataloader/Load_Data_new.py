"""The reference's bird's-eye-view loader (BEV/Dataloader/Load_Data_new.py) on the GPU, with the same public names and
signatures:

    from Dataloader.Load_Data_new import get_loader, get_homography, load_valid_set_file_all, write_lsq_results
    train_loader, valid_loader, valid_idx = get_loader(num_train, json_file, image_dir, gt_dir, flip_on, batch_size, shuffle,
                                                       num_workers, end_to_end, resize)
    for image, gt, params, idx, line_lst, horizon in train_loader:       # device tensors; idx on the CPU
        ...

A batch is the reference's collated tuple, element by element: image float32 [N,3,R,2R], gt int64 [N,1,R,2R], params
float32 [N,4,3] (Curve_parameters.json `poly_params`), idx int64 (CPU), line_lst int64 [N,4], horizon float32 [N,R], and for
validation batches index int64 (CPU), all bit-identical to the reference's.

The machinery is the TuSimple loader's (Dataloader/Load_Data_new.py of this package): the same device decoders, the same
cache of resized, unflipped samples, staging one batch ahead on a side stream, one flip draw np.random.uniform(0.0, 1.0) per
sample (validation samples included) in the main process when the batch is requested, the order of a torch DataLoader
with the reference's samplers, and the same end-of-epoch decoder check.  What is BEV's own:
  * Split: get_loader trims both splits to whole batches, and both use SubsetRandomSampler; no drop_last.
  * gt: classes 3 and 4 become 0; on a flip the map is mirrored and 1 and 2 are swapped (lf_loader_assemble_bev).
  * params and line_lst: per-row host tables for both flip states, built once with the reference's own expressions (the
    flip reorders the lanes [1, 0, 3, 2], negates, adds 1 to the constant term in float64, then casts to float32; the line
    types go through mirror_list; line_lst = lines[3:7] + 1 as int64, not clamped).
  * horizon: 1 above the first row of the resized map holding a value other than 0, 3 and 4 (the reference's
    gt.nonzero()[0, 1]).  lf_loader_label_rows records that row once per staged map; a flip does not move rows.

Deliberate differences:
  * flip_on=True: the reference calls F.hflip on the numpy label map, which torchvision rejects with TypeError, so its
    flipped training samples never load.  This loader does what the code after that call specifies: the map mirrored
    along its width, then 1 <-> 2 swapped, with the params and line types above.
  * A label map with no labelled pixel (the reference raises IndexError in __getitem__) raises ValueError naming the file
    at the end of the epoch that served it, from the end-of-epoch synchronisation, and again in every later epoch that
    serves it.  Its batch is yielded with a horizon of zeros.
  * A label row past the end of the params file or the line file raises IndexError when the dataset is built.
  * len() works (the reference's __len__ reads an attribute it never sets).
  * Files the device decoders do not support raise ValueError naming the file; there is no Pillow fallback.
Keyword-only extras: device, cache_bytes, expected_count (None: any number of files), line_file."""
import json
import os

import numpy as np
import torch
from torch.utils.data import Dataset

from lanedetection_end2end_b200 import _capi
from lanedetection_end2end_b200.Dataloader import Load_Data_new as _bp
from lanedetection_end2end_b200.Dataloader.Load_Data_new import (LaneLoader, _SampleStore, get_homography,  # noqa: F401
                                                                 homogenous_transformation, mirror_list)

NUM_LANES = _capi.LOADER_LANES
NUM_COEFFS = _capi.LOADER_BEV_COEFFS


# ---------------------------------------------------------------------------------------------------------------------
# host label tables (BEV/Dataloader/Load_Data_new.py:74-112 of the reference, per label row, for both flip states)

def _params(poly_params, flip):
    params = poly_params
    if flip:
        params = [params[1], params[0], params[3], params[2]]
        params = -np.array(params)
        params[:, -1] = 1 + params[:, -1]
    out = torch.from_numpy(np.array(params)).float().numpy()
    if out.shape != (NUM_LANES, NUM_COEFFS):
        raise ValueError("poly_params of shape %s; the loader needs %d lanes of %d coefficients" % (out.shape, NUM_LANES, NUM_COEFFS))
    return out


def _line_types(line_lst):
    return torch.from_numpy(np.array(np.array(line_lst[3:7]) + 1)).long().numpy()


def label_tables(params_file, line_file, rows):
    """Tables over the dataset positions whose label rows are `rows`: params float32 [2,P,4,3] and line int64 [2,P,4]
    (unflipped, flipped)."""
    P = len(rows)
    params = np.empty((2, P, NUM_LANES, NUM_COEFFS), np.float32)
    line = np.empty((2, P, NUM_LANES), np.int64)
    for p, r in enumerate(rows):
        for name, table in (("params", params_file), ("line", line_file)):
            if not 0 <= r < len(table):
                raise IndexError("label row %d is past the end of the %s file (%d rows)" % (r, name, len(table)))
        pp, ll = params_file[r]["poly_params"], line_file[r]["lines"]
        params[0, p], params[1, p] = _params(pp, False), _params(pp, True)
        line[0, p], line[1, p] = _line_types(ll), _line_types(mirror_list(ll))
    return {"params": params, "line": line}


# ---------------------------------------------------------------------------------------------------------------------
# dataset and loaders

class LaneDataset(Dataset):
    """Dataset with labeled lanes (the reference's BEV LaneDataset).  Indexing returns one sample as the reference's
    __getitem__ does (device tensors, idx and index as ints), drawing its flip; it checks the sample at once."""

    def __init__(self, end_to_end, valid_idx, json_file, image_dir, gt_dir, flip_on, resize, *, device=None, cache_bytes=None,
                 expected_count=2535, line_file="Labels/label_new.json"):
        self.image_dir = image_dir
        self.gt_dir = gt_dir
        self.flip_on = flip_on
        self.resize = resize
        self.params = _bp._json_lines(json_file)
        self.line_file = _bp._json_lines(line_file)
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
        self.tables = label_tables(self.params, self.line_file, self.rows)
        self._dev_tables = None
        self._store = _SampleStore([os.path.join(image_dir, n) for n in self.rgb_lst], [os.path.join(gt_dir, n) for n in self.gt_lst],
                                   resize, device, cache_bytes, label_rows=True)

    def __len__(self):
        return self.num_imgs

    _plan = _bp.LaneDataset._plan              # label rows, flip draws, validation index: the TuSimple loader's rules
    __getitem__ = _bp.LaneDataset.__getitem__

    def _assemble(self, plan, slots, staged):
        st = self._store
        if self._dev_tables is None:
            st._setup()
            self._dev_tables = {k: torch.from_numpy(np.ascontiguousarray(v)).to(st._dev) for k, v in self.tables.items()}
        stream, sample = st.assembly_begin(slots, plan.positions, [int(f) for f in plan.flips], staged)
        N, R, dev = len(slots), st.R, st._dev
        image = torch.empty(N, 3, R, 2 * R, dtype=torch.float32, device=dev)
        gt = torch.empty(N, 1, R, 2 * R, dtype=torch.int64, device=dev)
        params = torch.empty(N, NUM_LANES, NUM_COEFFS, dtype=torch.float32, device=dev)
        line = torch.empty(N, NUM_LANES, dtype=torch.int64, device=dev)
        horizon = torch.empty(N, R, dtype=torch.float32, device=dev)
        t, p = self._dev_tables, _capi.ptr
        _capi.call("lf_loader_assemble_bev", p(st.frames), p(st.maps), N, R, 2 * R, p(sample), len(self.rows), p(t["params"]),
                   p(t["line"]), p(st.first_row), p(image), p(gt), p(params), p(line), p(horizon), _capi.stream_ptr(),
                   nbytes=sum(o.numel() * o.element_size() for o in (image, gt, params, line, horizon)) + N * R * 2 * R * 4)
        st.assembly_end(stream, slots)
        idx = torch.tensor(plan.rows, dtype=torch.int64)
        if plan.index is not None:
            return image, gt, params, idx, line, horizon, torch.tensor(plan.index, dtype=torch.int64)
        return image, gt, params, idx, line, horizon


def get_loader(num_train, json_file, image_dir, gt_dir, flip_on, batch_size, shuffle, num_workers, end_to_end, resize,
               split_percentage=0.2, *, device=None, cache_bytes=None, expected_count=2535, line_file="Labels/label_new.json"):
    """Split the dataset into training and validation samples, each trimmed to whole batches, and make their loaders (one
    dataset, one cache)."""
    indices = list(range(num_train))
    split = int(np.floor(split_percentage * num_train))
    if shuffle is True:
        np.random.seed(num_train)
        np.random.shuffle(indices)
    train_idx, valid_idx = indices[split:], indices[:split]
    train_idx = train_idx[:len(train_idx) // batch_size * batch_size]
    valid_idx = valid_idx[:len(valid_idx) // batch_size * batch_size]
    train_sampler = torch.utils.data.sampler.SubsetRandomSampler(train_idx)
    valid_sampler = torch.utils.data.sampler.SubsetRandomSampler(valid_idx)
    transformed_dataset = LaneDataset(end_to_end=end_to_end, valid_idx=valid_idx, json_file=json_file, image_dir=image_dir,
                                      gt_dir=gt_dir, flip_on=flip_on, resize=resize, device=device, cache_bytes=cache_bytes,
                                      expected_count=expected_count, line_file=line_file)
    train_loader = LaneLoader(transformed_dataset, batch_size=batch_size, sampler=train_sampler, num_workers=num_workers)
    valid_loader = LaneLoader(transformed_dataset, batch_size=batch_size, sampler=valid_sampler, num_workers=num_workers)
    return train_loader, valid_loader, valid_idx


def load_valid_set_file_all(valid_idx, target_file, image_dir):
    """`target_file` = the rows of Labels/Curve_parameters.json of the validation samples, mapped through the string-sorted
    file names of `image_dir` (row int(name) - 1)."""
    labels_file = _bp._json_lines("Labels/Curve_parameters.json")
    target_idx = [int(i.split(".")[0]) for i in sorted(os.listdir(image_dir))]
    _bp._write_rows(target_file, labels_file, [target_idx[i] - 1 for i in valid_idx])


def write_lsq_results(src_file, dst_file, nclasses, all_branches_ready, horizon_on, resize, no_ortho, calc_intersection=False,
                      draw_image=False, path_test_set="../../../", test_phase=False):
    """Write `dst_file`: each row of `src_file` with its lanes replaced by the x coordinates (TuSimple pixels, -2 where
    absent) of its fitted curves `params`, sampled at its h_samples, through the bird's-eye-view homography unless
    `no_ortho`.  Points above max(210, the lane's first labelled y) -- or, with all_branches_ready and horizon_on, above
    the estimated horizon -- or below its last labelled y are -2.  With all_branches_ready, lanes 2 / 3 are skipped when
    line_id marks the outer left / right line absent; otherwise lanes without a labelled point are skipped.  The bytes the
    reference writes.  draw_image and calc_intersection are not supported (the reference's calc_intersection path calls
    a function it does not define)."""
    import cv2
    if draw_image:
        raise NotImplementedError("write_lsq_results(draw_image=True): drawing the predictions on test frames is not supported")
    if calc_intersection:
        raise NotImplementedError("write_lsq_results(calc_intersection=True) is not supported")
    factor = 640 / resize
    src = np.float32([[0.45, 0.3], [0.55, 0.3], [0.1, 1], [0.9, 1]])
    dst = np.float32([[0.45, 0.3], [0.55, 0.3], [0.45, 1], [0.55, 1]])
    M = cv2.getPerspectiveTransform(src, dst)
    M_inv = cv2.getPerspectiveTransform(dst, src)
    rows = _bp._json_lines(src_file)
    with open(dst_file, "w") as out:
        for row in rows:
            h_samples = row["h_samples"]
            y_orig = np.array(h_samples)
            y_d = (np.array(h_samples) - 80) / 639
            y_prime = (M[1][1] * y_d + M[1][2]) / (M[2][1] * y_d + M[2][2])
            y_eval = 1 - y_prime
            lanes_json = np.full((nclasses, len(h_samples)), -2)
            lanes, params, line_id = row["lanes"], row["params"], row["line_id"]
            absent = {2: line_id[0] == 0, 3: line_id[3] == 0}
            for j, pj in enumerate(params):
                lane = lanes if test_phase else lanes[j]
                h = [y for x, y in zip(lane, h_samples) if x != -2]
                if (absent.get(j, False) if all_branches_ready else not h):
                    continue
                minimum, maximum = (np.min(h), np.max(h)) if h else (250, 710)
                if all_branches_ready and horizon_on:
                    minimum = sum(row["horizon_est"]) * factor + 80
                a, b, c = [0] * (3 - len(pj)) + pj
                if not no_ortho:
                    x, _ = homogenous_transformation(M_inv, a * y_eval ** 2 + b * y_eval + c, y_prime)
                else:
                    y = 1 - y_d
                    x = a * y ** 2 + b * y + c
                x = np.int_(np.round(x * 1279))
                low = max(210, minimum)
                lanes_json[j] = [xi if low <= yi <= maximum else -2 for xi, yi in zip(x, y_orig)]
            row["run_time"] = 20
            row["lanes"] = lanes_json.tolist()
            json.dump(row, out)
            out.write("\n")
