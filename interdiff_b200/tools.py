"""Mirror of reference tools.py:11-76 point2point_signed on the sm_90a signed-nearest-neighbour
kernel (replaces the chamfer_distance CUDA extension the reference calls at tools.py:45-47)."""
import torch

from .engine import Engine

_ENGINES = {}


def _engine(device):
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("interdiff_b200.tools needs a CUDA (sm_90a) device: no CPU fallback")
    if device not in _ENGINES:
        _ENGINES[device] = Engine(device)
    return _ENGINES[device]


def point2point_signed(x, y, x_normals=None, y_normals=None, return_vector=False):
    """x (N,P1,3), y (N,P2,3) -> y2x_signed (N,P2), x2y_signed (N,P1), yidx_near, xidx_near [, y2x, x2y]"""
    if y.shape[0] != x.shape[0] or y.shape[2] != x.shape[2]:
        raise ValueError("y does not have the correct shape.")
    eng = _engine(x.device)
    y2x_signed, yidx, y2x = eng.signed_nn(y, x, x_normals)
    x2y_signed, xidx, x2y = eng.signed_nn(x, y, y_normals)
    if not return_vector:
        return y2x_signed, x2y_signed, yidx, xidx
    return y2x_signed, x2y_signed, yidx, xidx, y2x, x2y
