"""Mirror of reference data/tools.py:4-39 vertex_normals on the gather-based normals kernel."""
import numpy as np
import torch

from ..engine import Engine

_CACHE = {}


def vertex_normals(vertices, faces):
    """vertices (N,V,3); faces (N,Fc,3) -- the reference repeats one face table per frame
    (eval_smpl_short.py:110), so only faces[0] is read and every frame must share it."""
    assert vertices.ndimension() == 3 and faces.ndimension() == 3
    assert vertices.shape[0] == faces.shape[0] and vertices.shape[2] == 3 and faces.shape[2] == 3
    if vertices.device.type != "cuda":
        raise RuntimeError("interdiff_b200.data.tools needs a CUDA (sm_90a) device: no CPU fallback")
    V = vertices.shape[1]
    f0 = faces[0]
    key = (vertices.device, V, f0.data_ptr(), f0._version, tuple(f0.shape))
    eng = _CACHE.get(key)
    if eng is None:
        eng = Engine(vertices.device)
        z = np.zeros
        eng.load_body(dict(v_template=z((V, 3), np.float32), shapedirs=z((V, 3, 1), np.float32), posedirs=z((V, 3, 9), np.float32),
                           J_regressor=z((2, V), np.float32), weights=z((V, 2), np.float32), parents=np.array([0, 0]),
                           faces=f0.detach().cpu().numpy()))
        _CACHE.clear()
        _CACHE[key] = eng
    return eng.vertex_normals(vertices)
