"""lanedetection_end2end_b200 -- H100-native (sm_90a) hot path of
wvangansbeke/LaneDetection_End2End: ERFNet encoder/decoder -> per-lane weight maps ->
differentiable weighted least-squares layer -> loss on the curve coefficients.

Layout
  csrc/              hand-written CUDA kernels + the C ABI (include/lanefit_b200.h)
  _capi.py           ctypes binding of that ABI (no fallback if the .so is missing)
  ops_lsq.py, ops_net.py   autograd Functions over the ABI
  Networks/, Loss_crit.py  host-side mirror of the reference's module interface
                     (same names / arguments / state_dict keys), so that the
                     reference's main.py runs unchanged with this directory first on
                     sys.path (see INTEGRATION.md)
"""
__version__ = "0.1.0"
