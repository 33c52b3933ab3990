"""Birds_Eye_View_Loss/Loss_crit.py mirror: polynomial (:12-35), Area_Loss (:78-134) and MSE_Loss (:137-150) are shared
with the BP mirror, with fused_area_loss (the lanes' Area_Loss and the exact-area metric in one launch)."""
import importlib
import os
import sys

try:
    _L = importlib.import_module("lanedetection_end2end_b200.Loss_crit")
except ImportError:
    sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..", "..")))
    _L = importlib.import_module("lanedetection_end2end_b200.Loss_crit")

Area_Loss = _L.Area_Loss
MSE_Loss = _L.MSE_Loss
define_loss_crit = _L.define_loss_crit
polynomial = _L.polynomial
fused_area_loss = _L.fused_area_loss
