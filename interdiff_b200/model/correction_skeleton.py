"""Host-side mirror of reference model/correction_skeleton.py: ObjProjector (:8-135) for the skeleton model.
Parameters only (state_dict names of checkpoints/obj_skeleton.ckpt); sample() runs the projector kernel of
libinterdiff_b200.so (eval mode, BatchNorm folded, n_pre = 20, joint stack 9-64-32-64-9)."""
import torch
import torch.nn as nn

from ..engine import Engine
from .layers import ST_GCNN_layer


class ObjProjector(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.args = args
        self.n_pre = 20
        mk = lambda nodes, ver, chans: nn.ModuleList([ST_GCNN_layer(chans[i], chans[i + 1], [1, 1], 1, self.n_pre, nodes, args.dropout, version=ver)
                                                      for i in range(4)])
        self.st_gcnns_relative = mk(args.num_joints, 0, [9, 32, 16, 32, 9])
        self.st_gcnns = mk(1, 0, [9, 32, 16, 32, 9])
        self.st_gcnns_all = mk(args.num_joints + 1, 2, [9, 64, 32, 64, 9])

    def _signature(self):
        return tuple((k, v._version, v.data_ptr()) for k, v in self.state_dict().items())

    def load_into(self, eng):
        key = (id(self), self._signature())
        if getattr(eng, "_projector_owner", None) != key:
            eng.load_projector_skeleton(self.state_dict(), self.args.past_len, self.args.future_len, n_joints=self.args.num_joints)
            eng._projector_owner = key
        return eng

    def engine_for(self, device):
        engines = self.__dict__.setdefault("_engines", {})
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("interdiff_b200 skeleton ObjProjector runs on a CUDA (sm_90a) device only")
        if device not in engines:
            engines[device] = Engine(device)
        return self.load_into(engines[device])

    def sample(self, obj_angles, obj_trans, human_points):
        """obj_angles (T,B,4) quaternion xyzw, obj_trans (T,B,3), human_points (T,B,num_joints,3)
        -> (obj_angles_p (T,B,4) xyzw, obj_trans_p (T,B,3))   (reference :84-135, eval mode)."""
        if self.training:
            raise NotImplementedError("training mode is not on the sampling path")
        return self.engine_for(obj_angles.device).projector_sample_skeleton(obj_angles, obj_trans, human_points)

    def forward(self, obj_angles, obj_trans, human_points):
        """reference :69-80: (obj_angles_p, obj_trans_p, obj_angles_gt, obj_trans_gt)"""
        qp, tp = self.sample(obj_angles, obj_trans, human_points)
        return qp, tp, obj_angles.clone(), obj_trans.clone()
