"""Host-side mirror of reference model/correction_smpl.py: ObjProjector (:8-138).  Parameters
only; sample() runs the fused projector kernel of libinterdiff_b200.so (eval mode: argmax
hypothesis selection, BatchNorm folded)."""
import torch
import torch.nn as nn

from ..engine import Engine
from .layers import ST_GCNN_layer


class ObjProjector(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.args = args
        self.n_pre = args.dct
        chans = [9, 32, 16, 32, 9]
        mk = lambda nodes, ver: nn.ModuleList([ST_GCNN_layer(chans[i], chans[i + 1], [1, 1], 1, self.n_pre, nodes, args.dropout, version=ver)
                                               for i in range(4)])
        self.st_gcnns_relative = mk(args.num_verts, 0)
        self.st_gcnns = mk(1, 0)
        self.st_gcnns_all = mk(args.num_verts + 1, 2)

    def _signature(self):
        return tuple((k, v._version, v.data_ptr()) for k, v in self.state_dict().items())

    def load_into(self, eng):
        """Packs this module's weights into `eng` (shared with the denoiser for the fused loop)."""
        key = (id(self), self._signature())
        if getattr(eng, "_projector_owner", None) != key:     # tracked on the engine: projectors sharing one engine reload each other
            eng.load_projector(self.state_dict(), self.args.past_len, self.args.future_len, n_pre=self.n_pre, n_markers=self.args.num_verts)
            eng._projector_owner = key
        return eng

    def engine_for(self, device):
        engines = self.__dict__.setdefault("_engines", {})
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("interdiff_b200.ObjProjector runs on a CUDA (sm_90a) device only")
        if device not in engines:
            engines[device] = Engine(device)
        return self.load_into(engines[device])

    def sample(self, obj_angles, obj_trans, human_verts, contact, initialize=False):
        """obj_angles (T,B,6), obj_trans (T,B,3), human_verts (T,B,67,>=3), contact (B,67) -> (T,B,9)
        (reference :79-138, eval mode)."""
        if initialize or self.training:
            raise NotImplementedError("initialize=True / training-mode multinomial selection are training-time paths")
        eng = self.engine_for(obj_angles.device)
        return eng.projector_sample(obj_angles, obj_trans, human_verts[..., :3].contiguous(), contact)
