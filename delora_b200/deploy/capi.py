"""ctypes binding of the odometry workspaces of the C ABI (include/delora_b200.h): inference (`delora_odometry_pairs` /
`_push`), streams (`delora_odometry_streams_*`) and training (`delora_odometry_train_*`).

Each class holds one descriptor and one workspace, a torch uint8 tensor on the current device.  Every call runs on
torch's current stream at call time, checks its status with `_lib.check` and does not synchronise (except
`TrainingWorkspace.set_state`, whose inputs are temporaries).  Tensors are passed as device pointers, None where the
header allows NULL; the C side validates every argument, so nothing here repeats its checks."""
import ctypes

import torch

from .. import _lib, ops


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return None if t is None else t.data_ptr()


def train_params(config, lr, loss_flags=ops.LOSS_PO2PL | ops.LOSS_PL2PL, beta1=0.9, beta2=0.999, eps=1e-8):
    """delora_odometry_train_params: Adam's settings and the loss and normals' settings of a reference-style config."""
    nb = config["kitti"]["neighborhood_side_length"]
    return _lib.OdometryTrainParams(
        lr=lr, beta1=beta1, beta2=beta2, eps=eps, lambda_po2pl=config["lambda_po2pl"], loss_flags=loss_flags,
        nb_h=nb[0], nb_w=nb[1], epsilon_range=config["epsilon_range"],
        min_neighbors=config["min_num_points_in_neighborhood_to_determine_point_class"])


class _Workspace:
    SIZE_QUERY = None

    @classmethod
    def workspace_bytes(cls, desc):
        """The kind's size query; ValueError with the C side's message when it refuses the descriptor."""
        L = _lib.lib()
        nbytes = int(getattr(L, cls.SIZE_QUERY)(ctypes.byref(desc)))
        if nbytes < 0:
            raise ValueError(L.delora_last_error().decode())
        return nbytes

    def __init__(self, desc, workspace):
        self.desc = desc
        self._dp = ctypes.byref(desc)
        self._L = _lib.lib()
        nbytes = self.workspace_bytes(desc)
        if workspace is None:
            workspace = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
        elif workspace.numel() < nbytes:
            raise ValueError(f"the workspace has {workspace.numel()} bytes, the descriptor needs {nbytes}")
        self.workspace = workspace

    def _call(self, name, *args):
        """name(desc, *args, stream): every odometry entry point takes the descriptor first and the stream last."""
        _lib.check(getattr(self._L, name)(self._dp, *args, _stream()), name)


class InferenceWorkspace(_Workspace):
    """delora_odometry_workspace_bytes / _init / _load_weights / _pairs / _push."""
    SIZE_QUERY = "delora_odometry_workspace_bytes"

    def __init__(self, desc, weights, workspace=None):
        super().__init__(desc, workspace)
        self._call("delora_odometry_init", self.workspace.data_ptr())
        self.load_weights(weights)

    def load_weights(self, blob):
        self._call("delora_odometry_load_weights", blob.data_ptr(), self.workspace.data_ptr())

    def pairs(self, points, counts):
        """points [2B, 3, n_stride], counts [2B] -> (T [B, 4, 4], pooled [B, 512])."""
        b = points.shape[0] // 2
        t = torch.empty((b, 4, 4), dtype=torch.float32, device=self.workspace.device)
        pooled = torch.empty((b, 512), dtype=torch.float32, device=self.workspace.device)
        self._call("delora_odometry_pairs", points.data_ptr(), counts.data_ptr(), b, self.workspace.data_ptr(),
                   t.data_ptr(), pooled.data_ptr())
        return t, pooled

    def push(self, points, count, T):
        """One frame [1, 3, n_stride]; T [16] out, or None for a stream's first frame (project and cache only)."""
        self._call("delora_odometry_push", points.data_ptr(), count.data_ptr(), self.workspace.data_ptr(), _ptr(T))


class StreamsWorkspace(_Workspace):
    """delora_odometry_streams_*: S = desc.max_batch streams in one workspace."""
    SIZE_QUERY = "delora_odometry_streams_workspace_bytes"

    def __init__(self, desc, weights, workspace=None):
        super().__init__(desc, workspace)
        self._call("delora_odometry_streams_init", self.workspace.data_ptr())
        self._call("delora_odometry_streams_load_weights", weights.data_ptr(), self.workspace.data_ptr())

    def push(self, points, counts, active, T, valid):
        """points [S, 3, n_stride], counts [S], active [S] int32 or None (all active); T [S, 16] and valid [S] out."""
        self._call("delora_odometry_streams_push", points.data_ptr(), counts.data_ptr(), _ptr(active),
                   self.workspace.data_ptr(), T.data_ptr(), valid.data_ptr())

    def reset(self, mask):
        """Forget the previous frame of every stream with mask[s] != 0 (device int32 [S])."""
        self._call("delora_odometry_streams_reset", mask.data_ptr(), self.workspace.data_ptr())


class TrainingWorkspace(_Workspace):
    """delora_odometry_train_*: fp32 master weights, Adam's state and the step's buffers; `params` from train_params."""
    SIZE_QUERY = "delora_odometry_train_workspace_bytes"

    def __init__(self, desc, weights, params, workspace=None):
        super().__init__(desc, workspace)
        self._params = ctypes.byref(params)
        self.n = int(self._L.delora_odometry_weight_floats(self._dp))
        self._call("delora_odometry_train_init", weights.data_ptr(), self.workspace.data_ptr())

    def _floats(self):
        return torch.empty((self.n,), dtype=torch.float32, device=self.workspace.device)

    def step(self, points, counts, outputs=True):
        """One step on B = rows // 2 pairs -> (losses [B, 8], T [B, 4, 4], pooled [B, 512], grads [n]), or None
        without outputs."""
        b = points.shape[0] // 2
        out, ptrs = None, (None,) * 4
        if outputs:
            dev = self.workspace.device
            out = (torch.empty((b, ops.LOSS_ROW), dtype=torch.float32, device=dev),
                   torch.empty((b, 4, 4), dtype=torch.float32, device=dev),
                   torch.empty((b, 512), dtype=torch.float32, device=dev), self._floats())
            ptrs = tuple(t.data_ptr() for t in out)
        self._call("delora_odometry_train_step", self._params, points.data_ptr(), counts.data_ptr(), b,
                   self.workspace.data_ptr(), *ptrs)
        return out

    def weights(self):
        w = self._floats()
        self._call("delora_odometry_train_weights", self.workspace.data_ptr(), w.data_ptr())
        return w

    def get_state(self):
        """-> (weights, exp_avg, exp_avg_sq, step [1] int64) on the device."""
        st = (self._floats(), self._floats(), self._floats(),
              torch.empty((1,), dtype=torch.int64, device=self.workspace.device))
        self._call("delora_odometry_train_get_state", self.workspace.data_ptr(), *(t.data_ptr() for t in st))
        return st

    def set_state(self, weights, exp_avg, exp_avg_sq, step):
        """Array-likes of weight_floats floats each and the Adam step count; synchronises, as its inputs are copies."""
        dev = self.workspace.device
        step_t = torch.tensor([int(step)], dtype=torch.int64, device=dev)
        args = [torch.as_tensor(a, dtype=torch.float32).to(dev).contiguous() for a in (weights, exp_avg, exp_avg_sq)]
        self._call("delora_odometry_train_set_state", *(a.data_ptr() for a in args), step_t.data_ptr(),
                   self.workspace.data_ptr())
        torch.cuda.synchronize()
