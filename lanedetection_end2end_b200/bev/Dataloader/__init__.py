"""The reference's bird's-eye-view loader (BEV/Dataloader/), on the GPU: ``Load_Data_new`` has the reference's names and
signatures and yields collated device batches.  Importable as ``lanedetection_end2end_b200.bev.Dataloader`` or, with the
``bev`` directory first on sys.path the way the reference's BEV main.py imports it, as a top-level ``Dataloader``."""
import os
import sys

try:
    import lanedetection_end2end_b200  # noqa: F401
except ImportError:                     # top-level `Dataloader`: make the package importable
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))))
    import lanedetection_end2end_b200  # noqa: F401
