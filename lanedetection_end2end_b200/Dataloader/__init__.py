"""The reference's TuSimple loader (BP/Dataloader/), on the GPU: ``Load_Data_new`` has the reference's names and signatures
and yields collated device batches.  Importable as ``lanedetection_end2end_b200.Dataloader`` or, with the package directory
first on sys.path the way the reference's main.py imports it, as a top-level ``Dataloader``."""
import os
import sys

try:
    import lanedetection_end2end_b200  # noqa: F401
except ImportError:                     # top-level `Dataloader`: make the package importable
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
    import lanedetection_end2end_b200  # noqa: F401
