"""Host-side mirror of reference libsmpl/smplpytorch/pytorch/smpl_layer.py (SMPL_Layer :19-175).

Same constructor signature, buffer names (th_betas, th_shapedirs, th_posedirs, th_v_template,
th_J_regressor, th_weights, th_faces) and attributes (kintree_parents, num_joints); forward() runs
the fused SMPL-H LBS kernels of libinterdiff_b200.so.  The licensed SMPL-H .pkl is not shipped:
build the layer from arrays with SMPL_Layer.from_arrays(...) (a .pkl / .npz that unpickles to plain
arrays also works through the constructor).
"""
import os
import pickle

import numpy as np
import torch
from torch.nn import Module

from ....engine import Engine


def _load_arrays(path):
    if path.endswith(".npz"):
        with np.load(path, allow_pickle=True) as z:
            return {k: z[k] for k in z.files}
    with open(path, "rb") as f:
        d = pickle.load(f, encoding="latin1")  # needs chumpy only if the pkl holds chumpy arrays
    out = {}
    for k, v in d.items():
        out[k] = np.asarray(v.r) if hasattr(v, "r") else (v.toarray() if hasattr(v, "toarray") else v)
    return out


class SMPL_Layer(Module):
    __constants__ = ["kintree_parents", "gender", "center_idx", "num_joints"]

    def __init__(self, center_idx=None, gender="neutral", model_root="smpl/native/models", num_betas=300, hands=False, _arrays=None):
        super().__init__()
        self.center_idx, self.gender, self.model_root, self.hands = center_idx, gender, model_root, hands
        if _arrays is None:
            if hands:
                assert gender in ("male", "female"), "SMPL-H model only supports male or female, not {}".format(gender)
                self.model_path = os.path.join(model_root, f"SMPLH_{gender}.pkl")
            else:
                self.model_path = os.path.join(model_root, f"SMPL_{gender}.pkl")
            d = _load_arrays(self.model_path)
            parents = np.asarray(d["kintree_table"])[0].astype(np.int64)
            _arrays = dict(v_template=d["v_template"], shapedirs=np.asarray(d["shapedirs"])[:, :, :num_betas], posedirs=d["posedirs"],
                           J_regressor=d["J_regressor"], weights=d["weights"], faces=np.asarray(d["f"]).astype(np.int64),
                           parents=parents, betas=d.get("betas"))
        a = _arrays
        f32 = lambda x: torch.from_numpy(np.ascontiguousarray(np.asarray(x), dtype=np.float32))
        nb = np.asarray(a["shapedirs"]).shape[2]
        self.register_buffer("th_betas", f32(a["betas"]).reshape(1, -1) if a.get("betas") is not None else torch.zeros(1, nb))
        self.register_buffer("th_shapedirs", f32(a["shapedirs"]))
        self.register_buffer("th_posedirs", f32(a["posedirs"]))
        self.register_buffer("th_v_template", f32(a["v_template"]).unsqueeze(0))
        self.register_buffer("th_J_regressor", f32(a["J_regressor"]))
        self.register_buffer("th_weights", f32(a["weights"]))
        self.register_buffer("th_faces", torch.from_numpy(np.asarray(a["faces"]).astype(np.int64)))
        parents = [int(p) for p in np.asarray(a["parents"]).astype(np.int64)]
        parents[0] = -1  # stored as uint32(-1) in the pkl
        self.kintree_parents = parents
        self.num_joints = len(parents)

    @classmethod
    def from_arrays(cls, arrays, gender="male", hands=True, center_idx=None):
        return cls(center_idx=center_idx, gender=gender, hands=hands, _arrays=arrays)

    def arrays(self):
        return dict(v_template=self.th_v_template[0].cpu().numpy(), shapedirs=self.th_shapedirs.cpu().numpy(),
                    posedirs=self.th_posedirs.cpu().numpy(), J_regressor=self.th_J_regressor.cpu().numpy(),
                    weights=self.th_weights.cpu().numpy(), faces=self.th_faces.cpu().numpy(),
                    parents=np.asarray([max(p, 0) if i else 0 for i, p in enumerate(self.kintree_parents)], dtype=np.int64))

    def _signature(self):
        return tuple((k, v._version, v.data_ptr()) for k, v in self.state_dict().items())

    def load_into(self, eng):
        """The ENGINE remembers whose arrays it holds: two layers (male / female) alternating on one shared engine
        reload each other instead of silently running with the other's model."""
        key = (id(self), self._signature())
        if getattr(eng, "_body_owner", None) != key:
            eng.load_body(self.arrays())
            eng._body_owner = key
        return eng

    def engine_for(self, device):
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("interdiff_b200.SMPL_Layer runs on a CUDA (sm_90a) device only: no CPU fallback")
        engines = self.__dict__.setdefault("_engines", {})
        if device not in engines:
            engines[device] = Engine(device)
        return self.load_into(engines[device])

    def forward(self, th_pose_axisang, th_betas=None, th_trans=None, th_offsets=None, scale=1.0):
        """pose (F, J*3), betas (F, NB), trans (F, 3) -> (verts (F,V,3), joints (F,J,3), None, None).
        The reference also returns v_posed / naked, which no caller reads (eval_smpl_short.py:99,171)."""
        if th_offsets is not None or scale != 1.0:
            raise NotImplementedError("per-vertex offsets / scale are not used on the sampling path")
        F = th_pose_axisang.shape[0]
        dev = th_pose_axisang.device
        # reference :96-100: `th_betas is None or bool(torch.norm(th_betas) == 0)` switches to the layer's own template
        # betas (the default argument torch.zeros(1) lands here too); the norm test is a host sync upstream as well
        if th_betas is None or bool(torch.norm(th_betas) == 0):
            th_betas = self.th_betas.to(dev).expand(F, -1)
        elif th_betas.shape[0] == 1 and F > 1:
            th_betas = th_betas.expand(F, -1)
        if th_trans is None:
            th_trans = torch.zeros(F, 3, device=dev)
        if th_trans.shape[0] == 1 and F > 1:
            th_trans = th_trans.expand(F, -1)
        verts, jtr = self.engine_for(dev).lbs(th_pose_axisang, th_betas, th_trans)
        return verts, jtr, None, None
