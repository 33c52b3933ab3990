"""Host-side helpers the reference's drivers import from ``Networks.utils``
(BP/Networks/utils.py).  Only the pieces that are boundary inputs of the hot path are
real implementations here: the flag parser (:24-99, same flag names and defaults),
the homography (:104-121), weight init (:484-559), optimiser/scheduler factories
(:451-481) and the small bookkeeping classes main.py uses (:363-448).  Plotting helpers
(save_weightmap, draw_*) are host-side matplotlib I/O and out of scope (SURVEY.md 2).
"""
import argparse
import errno
import os
import sys

import numpy as np
import torch
import torch.nn.init as init
from torch.optim import lr_scheduler


def str2bool(argument):
    a = str(argument).lower()
    if a in ("yes", "true", "t", "y", "1"):
        return True
    if a in ("no", "false", "f", "n", "0"):
        return False
    raise argparse.ArgumentTypeError("Wrong argument in argparse, should be a boolean")


def _B(default):
    return dict(type=str2bool, nargs="?", const=True, default=default)


# (flag, kwargs) in the reference's order (BP/Networks/utils.py:26-98)
_FLAGS = [
    ("--dataset", dict(default="lane_detection")),
    ("--batch_size", dict(type=int, default=8)),
    ("--val_batch_size", dict(type=int, default=None)),
    ("--nepochs", dict(type=int, default=500)),
    ("--learning_rate", dict(type=float, default=1e-4)),
    ("--no_cuda", dict(action="store_true")),
    ("--nworkers", dict(type=int, default=8)),
    ("--no_dropout", dict(action="store_true")),
    ("--nclasses", dict(type=int, default=2, choices=[2, 4])),
    ("--crop_size", dict(type=int, default=80)),
    ("--resize", dict(type=int, default=256)),
    ("--mod", dict(type=str, default="erfnet")),
    ("--layers", dict(type=int, default=18)),
    ("--pool", _B(True)),
    ("--draw_testset", _B(False)),
    ("--pretrained", _B(False)),
    ("--pretrain_epochs", dict(type=int, default=20)),
    ("--skip_epochs", dict(type=int, default=10)),
    ("--channels_in", dict(type=int, default=3)),
    ("--norm", dict(type=str, default="batch")),
    ("--flip_on", _B(False)),
    ("--num_train", dict(type=int, default=3626)),
    ("--split_percentage", dict(type=float, default=0.2)),
    ("--test_mode", dict(action="store_true")),
    ("--start_epoch", dict(type=int, default=0)),
    ("--evaluate", dict(action="store_true")),
    ("--resume", dict(type=str, default="")),
    ("--optimizer", dict(type=str, default="adam")),
    ("--weight_init", dict(type=str, default="kaiming")),
    ("--weight_decay", dict(type=float, default=0)),
    ("--lr_decay", dict(action="store_true")),
    ("--niter", dict(type=int, default=50)),
    ("--niter_decay", dict(type=int, default=400)),
    ("--lr_policy", dict(default=None)),
    ("--lr_decay_iters", dict(type=int, default=30)),
    ("--clip_grad_norm", dict(type=int, default=0)),
    ("--order", dict(type=int, default=2)),
    ("--activation_layer", dict(type=str, default="square")),
    ("--reg_ls", dict(type=float, default=0)),
    ("--no_ortho", dict(action="store_true")),
    ("--mask_percentage", dict(type=float, default=0.3)),
    ("--use_cholesky", _B(False)),
    ("--activation_net", dict(type=str, default="relu")),
    ("--image_dir", dict(type=str, required=True)),
    ("--gt_dir", dict(type=str, required=True)),
    ("--test_dir", dict(type=str, default="/usr/data/tmp/Lane_Detection/TESTSET/")),
    ("--save_path", dict(type=str, default="Saved/")),
    ("--json_file", dict(type=str, default="Labels/Curve_parameters.json")),
    ("--weight_seg", dict(type=int, default=30)),
    ("--weight_class", dict(type=float, default=1)),
    ("--weight_fit", dict(type=float, default=1)),
    ("--loss_policy", dict(type=str, default="area")),
    ("--weight_funct", dict(type=str, default="none")),
    ("--end_to_end", _B(True)),
    ("--no_mapping", _B(False)),
    ("--learn_homography", _B(False)),
    ("--predict_homography", _B(False)),
    ("--predict_homography_corners", dict(type=str, default="destination", choices=["destination", "source"])),
    ("--seg_proxy", _B(False)),
    ("--weight_seg_proxy", dict(type=float, default=1.0)),
    ("--trapezium_mask", _B(False)),
    ("--gamma", dict(type=float, default=0.0)),
    ("--clas", _B(False)),
    ("--cudnn", _B(True)),
    ("--no_tb", _B(True)),
    ("--print_freq", dict(type=int, default=500)),
    ("--save_freq", dict(type=int, default=100)),
    ("--list", dict(type=int, nargs="+", default=[954, 2789])),
]


def define_args():
    parser = argparse.ArgumentParser(description="Lane_detection_all_objectives")
    for flag, kw in _FLAGS:
        parser.add_argument(flag, **kw)
    return parser


def _perspective_transform(src, dst):
    """4-point homography (h33 = 1) -- cv2.getPerspectiveTransform when OpenCV is
    importable (bit-identical to what the reference computes with the same OpenCV),
    else the same 8x8 DLT system solved with numpy."""
    try:
        import cv2
        return cv2.getPerspectiveTransform(np.float32(src), np.float32(dst))
    except ImportError:
        s = np.asarray(src, np.float64)
        t = np.asarray(dst, np.float64)
        A, b = np.zeros((8, 8)), np.zeros(8)
        for i in range(4):
            (x, y), (X, Y) = s[i], t[i]
            A[i] = [x, y, 1, 0, 0, 0, -x * X, -y * X]
            A[i + 4] = [0, 0, 0, x, y, 1, -x * Y, -y * Y]
            b[i], b[i + 4] = X, Y
        return np.append(np.linalg.solve(A, b), 1.0).reshape(3, 3)


def get_homography(resize=256, no_mapping=False):
    """Image -> bird's-eye-view homography and its inverse (BP/Networks/utils.py:104-121):
    a trapezoid (2 %..97 % of the width at the bottom row, 45 %..55 % at 20 % height) is
    mapped onto the 45 %..55 % column band."""
    if no_mapping:
        return np.identity(3), np.identity(3)
    w = 2 * resize
    top, bottom = 0.20 * resize, resize - 1
    src = np.float32([[0.45 * w, top], [0.55 * w, top], [0.02 * w, bottom], [0.97 * w, bottom]])
    dst = np.float32([[0.45 * w, top], [0.55 * w, top], [0.45 * w, bottom], [0.55 * w, bottom]])
    return _perspective_transform(src, dst), _perspective_transform(dst, src)


def save_weightmap(*args, **kwargs):
    """Plotting helper of the reference (BP/Networks/utils.py:127-187): host-side
    matplotlib I/O, out of the hot-path scope.  No-op here."""
    return None


def first_run(save_path):
    txt_file = os.path.join(save_path, "first_run.txt")
    if not os.path.exists(txt_file):
        open(txt_file, "w").close()
        return ""
    return open(txt_file).read() or ""


def mkdir_if_missing(directory):
    try:
        os.makedirs(directory, exist_ok=True)
    except OSError as e:  # pragma: no cover
        if e.errno != errno.EEXIST:
            raise


class Logger(object):
    """Tee stdout to a file (BP/Networks/utils.py:395-430)."""

    def __init__(self, fpath=None):
        self.console = sys.stdout
        self.file = None
        if fpath is not None:
            mkdir_if_missing(os.path.dirname(fpath))
            self.file = open(fpath, "w")

    def write(self, msg):
        self.console.write(msg)
        if self.file is not None:
            self.file.write(msg)

    def flush(self):
        self.console.flush()
        if self.file is not None:
            self.file.flush()
            os.fsync(self.file.fileno())

    def close(self):
        if self.file is not None:
            self.file.close()
            self.file = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class AverageMeter(object):
    def __init__(self):
        self.reset()

    def reset(self):
        self.val = self.avg = self.sum = self.count = 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def define_optim(optim, params, lr, weight_decay, fused=None, per_param_step=False, max_grad_norm=None):
    """torch.optim's Adam / SGD / RMSprop (BP/Networks/utils.py:451-461), or with ``fused`` the same update as one launch
    of the library's kernel (lanedetection_end2end_b200.optim.FusedOptimizer, CUDA-graph capturable, same state_dict
    format).  fused=None reads LANEFIT_FUSED_OPTIM (default 0: the torch optimizer), so the reference's main.py can opt in
    without edits.  ``per_param_step``: the FusedOptimizer keeps one step count per parameter, as torch.optim does (needed
    by --pretrained, whose phases train different parameter sets); the torch optimizers always do, so it changes nothing
    for them.  ``max_grad_norm``: the FusedOptimizer clips the gradients by their global L2 norm inside its update (see
    FusedOptimizer); the torch optimizers ignore it (clip with torch.nn.utils.clip_grad_norm_ before their step())."""
    if fused is None:
        fused = os.environ.get("LANEFIT_FUSED_OPTIM", "0") != "0"
    if fused and optim in ("adam", "sgd", "rmsprop"):
        from ._pkg import submodule
        return submodule("optim").FusedOptimizer(params, optim, lr, weight_decay, per_param_step=per_param_step,
                                                 max_grad_norm=max_grad_norm)
    if optim == "adam":
        return torch.optim.Adam(params, lr=lr, weight_decay=weight_decay)
    if optim == "sgd":
        return torch.optim.SGD(params, lr=lr, momentum=0.9, weight_decay=weight_decay)
    if optim == "rmsprop":
        return torch.optim.RMSprop(params, lr=lr, momentum=0.9, weight_decay=weight_decay)
    raise KeyError("The requested optimizer: {} is not implemented".format(optim))


def define_scheduler(optimizer, args):
    if args.lr_policy == "lambda":
        return lr_scheduler.LambdaLR(
            optimizer, lr_lambda=lambda epoch: 1.0 - max(0, epoch + 1 - args.niter) / float(args.niter_decay + 1))
    if args.lr_policy == "step":
        return lr_scheduler.StepLR(optimizer, step_size=args.lr_decay_iters, gamma=args.gamma)
    if args.lr_policy == "plateau":
        return lr_scheduler.ReduceLROnPlateau(optimizer, mode="min", factor=args.gamma, threshold=0.0001,
                                              patience=args.lr_decay_iters)
    if args.lr_policy == "none":
        return None
    return NotImplementedError("learning rate policy [%s] is not implemented", args.lr_policy)


def _init_module(m, conv_init):
    """One rule for every scheme (BP/Networks/utils.py:498-559): Conv*/Linear weights by
    ``conv_init``, their biases zero; BatchNorm2d weight ~ N(1, 0.02), bias 0."""
    name = m.__class__.__name__
    if getattr(m, "zero_init", False):
        # the predicted homography's last layer (homography.SpatialTransformer.fully_connected2) stays at zero so that a
        # new model starts from the fixed warp; the reference's kaiming init would re-draw it
        m.weight.data.zero_()
        m.bias.data.zero_()
    elif "Conv" in name or "Linear" in name or name in ("DownConv", "FactorisedConv"):
        w = getattr(m, "weight", None)
        if w is not None:
            conv_init(w.data)
            if getattr(m, "bias", None) is not None:
                m.bias.data.zero_()
    elif "BatchNorm2d" in name:
        init.normal_(m.weight.data, 1.0, 0.02)
        init.constant_(m.bias.data, 0.0)


_INIT = {
    "normal": lambda w: init.normal_(w, 0.0, 0.02),
    "xavier": lambda w: init.xavier_normal_(w, gain=0.02),
    "kaiming": lambda w: init.kaiming_normal_(w, a=0, mode="fan_in", nonlinearity="relu"),
    "orthogonal": lambda w: init.orthogonal_(w, gain=1),
}


def define_init_weights(model, init_w="normal", activation="relu"):
    print("Init weights in network with [{}]".format(init_w))
    if init_w not in _INIT:
        raise NotImplementedError("initialization method [{}] is not implemented".format(init_w))
    model.apply(lambda m: _init_module(m, _INIT[init_w]))
