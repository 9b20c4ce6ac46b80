"""ctypes binding of the odometry workspaces of the C ABI (include/delora_b200.h): inference (`delora_odometry_pairs` /
`_pairs_normalized` / `_push`), streams (`delora_odometry_streams_*`, with the per-frame ICP residual
`delora_odometry_streams_residual_*` / `_push_residual`, for normalised models
`delora_odometry_streams_normalized_*` / `_push_normalized`, and on the reference's two-resolution recipe
`delora_odometry_streams_pre_*` / `_push_pre`) and training (`delora_odometry_train_*`, and
`delora_odometry_train_step_group` for several workspaces stepped as one data-parallel group,
`delora_odometry_train_geometries_*` / `_use_geometry` for one workspace shared by several sensor geometries), and
streams that adapt the model while serving it (`delora_odometry_streams_adapt_*` / `_push_adapt`, and
`delora_odometry_streams_push_adapt_group` for one model adapted from the streams of several workspaces).

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


def _objective(config, loss_flags):
    """(loss_flags, lambda_po2pl): the caller's flags with the config's lambda_po2pl, or with loss_flags None the
    objective the config names (export.objective_from_config, the objective a .dlw / .dlt records)."""
    from . import export
    if loss_flags is None:
        return export.objective_from_config(config)
    return loss_flags, config["lambda_po2pl"]


def train_params(config, lr, loss_flags=None, beta1=0.9, beta2=0.999, eps=1e-8):
    """delora_odometry_train_params: Adam's settings and the loss and normals' settings of a reference-style config.
    loss_flags: the ICP loss bits, or None for the objective the config names (po2po_alone included).
    normalization_scaling: True adds DELORA_TRAIN_NORMALIZATION_SCALING (the step then needs a descriptor with
    w_pre > 0, and refuses w_pre = 0); use_dropout: True adds DELORA_TRAIN_DROPOUT."""
    nb = config["kitti"]["neighborhood_side_length"]
    loss_flags, lam = _objective(config, loss_flags)
    if config.get("normalization_scaling", False):
        loss_flags |= ops.TRAIN_NORMALIZATION_SCALING
    if config.get("use_dropout", False):
        loss_flags |= ops.TRAIN_DROPOUT
    return _lib.OdometryTrainParams(
        lr=lr, beta1=beta1, beta2=beta2, eps=eps, lambda_po2pl=lam, loss_flags=loss_flags,
        nb_h=nb[0], nb_w=nb[1], epsilon_range=config["epsilon_range"],
        min_neighbors=config["min_num_points_in_neighborhood_to_determine_point_class"])


def residual_params(config, loss_flags=None):
    """delora_odometry_residual_params: the loss and normals' settings of a reference-style config; loss_flags as for
    train_params."""
    nb = config["kitti"]["neighborhood_side_length"]
    loss_flags, lam = _objective(config, loss_flags)
    return _lib.OdometryResidualParams(
        lambda_po2pl=lam, loss_flags=loss_flags, nb_h=nb[0], nb_w=nb[1],
        epsilon_range=config["epsilon_range"],
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
    """delora_odometry_workspace_bytes / _init / _load_weights / _pairs / _pairs_normalized / _push."""
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

    def pairs_normalized(self, points, counts):
        """A model trained with normalization_scaling: points [2B, 3, n_stride], counts [2B] -> (T [B, 4, 4] with the
        translation in metres, pooled [B, 512], factor [B])."""
        b = points.shape[0] // 2
        dev = self.workspace.device
        t = torch.empty((b, 4, 4), dtype=torch.float32, device=dev)
        pooled = torch.empty((b, 512), dtype=torch.float32, device=dev)
        factor = torch.empty((b,), dtype=torch.float32, device=dev)
        self._call("delora_odometry_pairs_normalized", points.data_ptr(), counts.data_ptr(), b,
                   self.workspace.data_ptr(), t.data_ptr(), pooled.data_ptr(), factor.data_ptr())
        return t, pooled, factor

    def push(self, points, count, T):
        """One frame [1, 3, n_stride]; T [16] out, or None for a stream's first frame (project and cache only)."""
        self._call("delora_odometry_push", points.data_ptr(), count.data_ptr(), self.workspace.data_ptr(), _ptr(T))


class StreamsWorkspace(_Workspace):
    """delora_odometry_streams_*: S = desc.max_batch streams in one workspace."""
    SIZE_QUERY = "delora_odometry_streams_workspace_bytes"
    INIT = "delora_odometry_streams_init"

    def __init__(self, desc, weights, workspace=None):
        super().__init__(desc, workspace)
        self._call(self.INIT, self.workspace.data_ptr())
        self.load_weights(weights)

    def load_weights(self, blob):
        """delora_odometry_streams_load_weights: replace the weights; every stream keeps its previous frame."""
        self._call("delora_odometry_streams_load_weights", blob.data_ptr(), self.workspace.data_ptr())

    def push(self, points, counts, active, T, valid):
        """points [S, 3, n_stride], counts [S], active [S] int32 or None (all active); T [S, 16] and valid [S] out."""
        self._call("delora_odometry_streams_push", points.data_ptr(), counts.data_ptr(), _ptr(active),
                   self.workspace.data_ptr(), T.data_ptr(), valid.data_ptr())

    def reset(self, mask):
        """Forget the previous frame of every stream with mask[s] != 0 (device int32 [S])."""
        self._call("delora_odometry_streams_reset", mask.data_ptr(), self.workspace.data_ptr())


class ResidualStreamsWorkspace(StreamsWorkspace):
    """delora_odometry_streams_residual_* on the streams layout with the residual's sections appended: `push` also
    writes each stream's ICP loss row; `params` from residual_params.  load_weights / reset are the streams calls."""
    SIZE_QUERY = "delora_odometry_streams_residual_workspace_bytes"
    INIT = "delora_odometry_streams_residual_init"

    def __init__(self, desc, weights, params, workspace=None):
        super().__init__(desc, weights, workspace)
        self._params = ctypes.byref(params)

    def push(self, points, counts, active, T, valid, losses):
        """StreamsWorkspace.push plus losses [S, LOSS_ROW] out: the ICP row of every valid stream, zeros elsewhere."""
        self._call("delora_odometry_streams_push_residual", self._params, points.data_ptr(), counts.data_ptr(),
                   _ptr(active), self.workspace.data_ptr(), T.data_ptr(), valid.data_ptr(), losses.data_ptr())


class InformationStreamsWorkspace(ResidualStreamsWorkspace):
    """delora_odometry_streams_info_* on the residual layout with the information section appended: `push` also writes
    each stream's information row (the Gauss-Newton information of the residual's objective at T).  load_weights /
    reset are the streams calls."""
    SIZE_QUERY = "delora_odometry_streams_info_workspace_bytes"
    INIT = "delora_odometry_streams_info_init"

    def push(self, points, counts, active, T, valid, losses, info):
        """ResidualStreamsWorkspace.push plus info [S, INFO_ROW] out: the information row of every valid stream, zeros
        elsewhere."""
        self._call("delora_odometry_streams_push_info", self._params, points.data_ptr(), counts.data_ptr(),
                   _ptr(active), self.workspace.data_ptr(), T.data_ptr(), valid.data_ptr(), losses.data_ptr(),
                   info.data_ptr())


class NormalizedStreamsWorkspace(StreamsWorkspace):
    """delora_odometry_streams_normalized_* for a model trained with normalization_scaling, on the streams layout with
    the normalised sections appended: `push` also writes each pair's factor.  load_weights / reset are the streams
    calls."""
    SIZE_QUERY = "delora_odometry_streams_normalized_workspace_bytes"
    INIT = "delora_odometry_streams_normalized_init"

    def push(self, points, counts, active, T, valid, factor):
        """StreamsWorkspace.push plus factor [S] out: the factor of every valid stream's pair, 0 elsewhere; T's
        translation is in the points' units."""
        self._call("delora_odometry_streams_push_normalized", points.data_ptr(), counts.data_ptr(), _ptr(active),
                   self.workspace.data_ptr(), T.data_ptr(), valid.data_ptr(), factor.data_ptr())


class PreStreamsWorkspace(StreamsWorkspace):
    """delora_odometry_streams_pre_* (the descriptor needs w_pre > 0): the streams served on the reference's
    two-resolution recipe, with the training step's ICP residual; `params` from residual_params, with
    TRAIN_NORMALIZATION_SCALING in its loss_flags for a normalised model.  load_weights / reset are the streams calls."""
    SIZE_QUERY = "delora_odometry_streams_pre_workspace_bytes"
    INIT = "delora_odometry_streams_pre_init"

    def __init__(self, desc, weights, params, workspace=None):
        super().__init__(desc, weights, workspace)
        self._params = ctypes.byref(params)

    def push(self, points, counts, active, T, valid, losses, factor=None):
        """StreamsWorkspace.push plus losses [S, LOSS_ROW] out (the ICP row of every valid stream, zeros elsewhere) and,
        for a normalised model only, factor [S] out (the pair's factor where valid, 0 elsewhere)."""
        self._call("delora_odometry_streams_push_pre", self._params, points.data_ptr(), counts.data_ptr(), _ptr(active),
                   self.workspace.data_ptr(), T.data_ptr(), valid.data_ptr(), losses.data_ptr(), _ptr(factor))


class PreInformationStreamsWorkspace(PreStreamsWorkspace):
    """delora_odometry_streams_pre_info_* on the recipe layout with the information section appended: `push` also writes
    each stream's information row at T, in the metres and radians of T for normalised models too.  load_weights / reset
    are the streams calls."""
    SIZE_QUERY = "delora_odometry_streams_pre_info_workspace_bytes"
    INIT = "delora_odometry_streams_pre_info_init"

    def push(self, points, counts, active, T, valid, losses, info, factor=None):
        """PreStreamsWorkspace.push plus info [S, INFO_ROW] out: the information row of every valid stream, zeros
        elsewhere."""
        self._call("delora_odometry_streams_push_pre_info", self._params, points.data_ptr(), counts.data_ptr(),
                   _ptr(active), self.workspace.data_ptr(), T.data_ptr(), valid.data_ptr(), losses.data_ptr(),
                   _ptr(factor), info.data_ptr())


class TrainingWorkspace(_Workspace):
    """delora_odometry_train_*: fp32 master weights, Adam's state and the step's buffers; `params` from train_params."""
    SIZE_QUERY = "delora_odometry_train_workspace_bytes"

    def __init__(self, desc, weights, params, workspace=None):
        super().__init__(desc, workspace)
        self._params = ctypes.byref(params)
        self.n = int(self._L.delora_odometry_weight_floats(self._dp))
        self._init(weights)

    def _init(self, weights):
        self._call("delora_odometry_train_init", weights.data_ptr(), self.workspace.data_ptr())

    def _floats(self):
        return torch.empty((self.n,), dtype=torch.float32, device=self.workspace.device)

    def _step_outputs(self, b, outputs):
        if not outputs:
            return None, (None,) * 4
        dev = self.workspace.device
        out = (torch.empty((b, ops.LOSS_ROW), dtype=torch.float32, device=dev),
               torch.empty((b, 4, 4), dtype=torch.float32, device=dev),
               torch.empty((b, 512), dtype=torch.float32, device=dev), self._floats())
        return out, tuple(t.data_ptr() for t in out)

    def step(self, points, counts, outputs=True):
        """One step on B = rows // 2 pairs -> (losses [B, 8], T [B, 4, 4], pooled [B, 512], grads [n]), or None
        without outputs.  Normalised models: losses[:, 6] is each pair's factor and T's translation is in metres."""
        b = points.shape[0] // 2
        out, ptrs = self._step_outputs(b, outputs)
        self._call("delora_odometry_train_step", self._params, points.data_ptr(), counts.data_ptr(), b,
                   self.workspace.data_ptr(), *ptrs)
        return out

    def step_group(self, group, points, counts, outputs=True):
        """delora_odometry_train_step_group with `group` (a _lib.OdometryTrainGroup whose rank is this workspace):
        step's outputs, grads being the gradient averaged over the group."""
        b = points.shape[0] // 2
        out, ptrs = self._step_outputs(b, outputs)
        self._call("delora_odometry_train_step_group", self._params, ctypes.byref(group), points.data_ptr(),
                   counts.data_ptr(), b, self.workspace.data_ptr(), *ptrs)
        return out

    def eval(self, points, counts):
        """delora_odometry_train_eval on B = rows // 2 pairs -> (losses [B, 8], T [B, 4, 4], pooled [B, 512]): the ICP
        losses of the current weights, nothing updated; dropout is the identity."""
        b = points.shape[0] // 2
        dev = self.workspace.device
        out = (torch.empty((b, ops.LOSS_ROW), dtype=torch.float32, device=dev),
               torch.empty((b, 4, 4), dtype=torch.float32, device=dev),
               torch.empty((b, 512), dtype=torch.float32, device=dev))
        self._call("delora_odometry_train_eval", self._params, points.data_ptr(), counts.data_ptr(), b,
                   self.workspace.data_ptr(), *(t.data_ptr() for t in out))
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

    def set_dropout_seed(self, seed):
        """The seed of the dropout masks (DELORA_TRAIN_DROPOUT steps); 0 after construction.  Only launches."""
        self._call("delora_odometry_train_set_dropout_seed", int(seed) & 0xFFFFFFFFFFFFFFFF, self.workspace.data_ptr())

    def set_state(self, weights, exp_avg, exp_avg_sq, step):
        """Array-likes of weight_floats floats each and the Adam step count; synchronises, as its inputs are copies."""
        dev = self.workspace.device
        step_t = torch.tensor([int(step)], dtype=torch.int64, device=dev)
        args = [torch.as_tensor(a, dtype=torch.float32).to(dev).contiguous() for a in (weights, exp_avg, exp_avg_sq)]
        self._call("delora_odometry_train_set_state", *(a.data_ptr() for a in args), step_t.data_ptr(),
                   self.workspace.data_ptr())
        torch.cuda.synchronize()


class AdaptiveStreamsWorkspace(TrainingWorkspace):
    """delora_odometry_streams_adapt_*: S = desc.max_batch streams served from a training workspace that takes the
    training step on the pairs it has just served.  Every TrainingWorkspace call works on it (weights, get_state /
    set_state, eval) and leaves the stream section alone; `params` from train_params (without use_dropout)."""
    SIZE_QUERY = "delora_odometry_streams_adapt_workspace_bytes"

    def _init(self, weights):
        self._call("delora_odometry_streams_adapt_init", weights.data_ptr(), self.workspace.data_ptr())

    def push(self, points, counts, active, T, valid, losses, update=True):
        """points [S, 3, n_stride], counts [S], active [S] int32 or None (all active); T [S, 16], valid [S] and losses
        [S, LOSS_ROW] out, as for PreStreamsWorkspace.push (T of the weights before this tick's update).  update: then
        one Adam step on the mean objective of the valid pairs (none without a valid pair)."""
        self._call("delora_odometry_streams_push_adapt", self._params, 1 if update else 0, points.data_ptr(),
                   counts.data_ptr(), _ptr(active), self.workspace.data_ptr(), T.data_ptr(), valid.data_ptr(),
                   losses.data_ptr())

    def reset(self, mask):
        """Forget the previous frame of every stream with mask[s] != 0 (device int32 [S])."""
        self._call("delora_odometry_streams_adapt_reset", mask.data_ptr(), self.workspace.data_ptr())


class GeometriesTrainingWorkspace(TrainingWorkspace):
    """delora_odometry_train_geometries_*: one training workspace shared by several sensor geometries (descriptors with
    the same model fields and W parity).  `use(g)` re-arms it for descs[g]; every TrainingWorkspace call after it runs
    with descs[g].  Armed for descs[0] after construction."""

    @staticmethod
    def shared_bytes(descs):
        """delora_odometry_train_geometries_workspace_bytes; ValueError with the C side's message when it refuses."""
        L = _lib.lib()
        arr = (_lib.OdometryDesc * len(descs))(*descs)
        nbytes = int(L.delora_odometry_train_geometries_workspace_bytes(arr, len(arr)))
        if nbytes < 0:
            raise ValueError(L.delora_last_error().decode())
        return nbytes

    def __init__(self, descs, weights, params, workspace=None):
        self.descs = (_lib.OdometryDesc * len(descs))(*descs)
        nbytes = self.shared_bytes(self.descs)
        if workspace is None:
            workspace = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
        elif workspace.numel() < nbytes:
            raise ValueError(f"the workspace has {workspace.numel()} bytes, the geometries need {nbytes}")
        self.geometry = 0
        super().__init__(self.descs[0], weights, params, workspace)

    def _init(self, weights):
        name = "delora_odometry_train_geometries_init"
        _lib.check(getattr(self._L, name)(self.descs, len(self.descs), weights.data_ptr(), self.workspace.data_ptr(),
                                          _stream()), name)

    def use(self, g):
        """delora_odometry_train_use_geometry: re-arm the geometry section for descs[g] (only launches)."""
        name = "delora_odometry_train_use_geometry"
        _lib.check(getattr(self._L, name)(self.descs, len(self.descs), int(g), self.workspace.data_ptr(), _stream()),
                   name)
        self.geometry = int(g)
        self.desc = self.descs[self.geometry]
        self._dp = ctypes.byref(self.desc)


class GeometriesAdaptingStreamsWorkspace(TrainingWorkspace):
    """delora_odometry_streams_adapt_geometries_*: one model adapted from the streams of several sensor geometries in
    one workspace.  Geometry g serves descs[g].max_batch streams; streams are numbered in geometry order
    (`n_streams` in all).  Every TrainingWorkspace call runs with descs[0] (weights, get_state / set_state) and leaves
    the stream sections alone; `params` from train_params (without use_dropout)."""
    GEOMETRIES_SIZE_QUERY = "delora_odometry_streams_adapt_geometries_workspace_bytes"

    @classmethod
    def shared_bytes(cls, descs):
        """The kind's size query over descs; ValueError with the C side's message when it refuses."""
        L = _lib.lib()
        arr = (_lib.OdometryDesc * len(descs))(*descs)
        nbytes = int(getattr(L, cls.GEOMETRIES_SIZE_QUERY)(arr, len(arr)))
        if nbytes < 0:
            raise ValueError(L.delora_last_error().decode())
        return nbytes

    def __init__(self, descs, weights, params, workspace=None):
        self.descs = (_lib.OdometryDesc * len(descs))(*descs)
        nbytes = self.shared_bytes(self.descs)
        if workspace is None:
            workspace = torch.empty((nbytes,), dtype=torch.uint8, device="cuda")
        elif workspace.numel() < nbytes:
            raise ValueError(f"the workspace has {workspace.numel()} bytes, the geometries need {nbytes}")
        self.streams = [int(d.max_batch) for d in self.descs]
        self.n_streams = sum(self.streams)
        super().__init__(self.descs[0], weights, params, workspace)

    def _geometries_call(self, name, *args):
        _lib.check(getattr(self._L, name)(self.descs, len(self.descs), *args, _stream()), name)

    def _init(self, weights):
        self._geometries_call("delora_odometry_streams_adapt_geometries_init", weights.data_ptr(),
                              self.workspace.data_ptr())

    def push(self, points, counts, active, T, valid, losses, update=True):
        """points / counts: one device tensor per geometry, [S_g, 3, descs[g].n_stride] and [S_g]; active [n_streams]
        int32 or None (all active); T [n_streams, 16], valid [n_streams] and losses [n_streams, LOSS_ROW] out, as for
        AdaptiveStreamsWorkspace.push.  update: then one Adam step on the mean objective of every geometry's valid
        pairs."""
        n = len(self.descs)
        pts = (ctypes.c_void_p * n)(*(p.data_ptr() for p in points))
        cnt = (ctypes.c_void_p * n)(*(c.data_ptr() for c in counts))
        self._geometries_call("delora_odometry_streams_push_adapt_geometries", self._params,
                              1 if update else 0, pts, cnt, _ptr(active), self.workspace.data_ptr(), T.data_ptr(),
                              valid.data_ptr(), losses.data_ptr())

    def reset(self, mask):
        """Forget the previous frame of every stream with mask[s] != 0 (device int32 [n_streams])."""
        self._geometries_call("delora_odometry_streams_adapt_geometries_reset", mask.data_ptr(),
                              self.workspace.data_ptr())


class GeometriesAdaptingInformationStreamsWorkspace(GeometriesAdaptingStreamsWorkspace):
    """delora_odometry_streams_adapt_geometries_info_*: the geometries layout of the adapting streams with the
    information section appended; every GeometriesAdaptingStreamsWorkspace call works on it.  `push` takes info
    [n_streams, INFO_ROW] out after losses: the information row at the served T (before the tick's update) of every
    valid stream, in the metres and radians of T for normalised models too; zeros elsewhere."""
    GEOMETRIES_SIZE_QUERY = "delora_odometry_streams_adapt_geometries_info_workspace_bytes"

    def push(self, points, counts, active, T, valid, losses, info, update=True):
        n = len(self.descs)
        pts = (ctypes.c_void_p * n)(*(p.data_ptr() for p in points))
        cnt = (ctypes.c_void_p * n)(*(c.data_ptr() for c in counts))
        self._geometries_call("delora_odometry_streams_push_adapt_geometries_info", self._params,
                              1 if update else 0, pts, cnt, _ptr(active), self.workspace.data_ptr(), T.data_ptr(),
                              valid.data_ptr(), losses.data_ptr(), info.data_ptr())


class TrainingGroup:
    """The delora_odometry_train_group of each of N TrainingWorkspaces (same descriptor and state), on N devices with
    peer access enabled between them or all on one device: the flag words and status word of every rank (on its
    workspace's device, zeroed), a side stream and the six events per rank, unicast path.  `groups[r]` is rank r's
    descriptor; `step(r, ...)` runs rank r's group step on the current stream of its device."""

    def __init__(self, workspaces, n_ctas=8, n_threads=128):
        L = _lib.lib()
        world = len(workspaces)
        self.workspaces = workspaces
        self.flags = [torch.zeros(L.delora_grad_allreduce_flag_words(), dtype=torch.int32, device=w.workspace.device)
                      for w in workspaces]
        self.status = [torch.zeros(1, dtype=torch.int32, device=w.workspace.device) for w in workspaces]
        self.side_streams, self.events, self.groups = [], [], []
        for r, w in enumerate(workspaces):
            dev = w.workspace.device
            side = torch.cuda.Stream(device=dev)
            events = [torch.cuda.Event() for _ in range(_lib.TRAIN_GROUP_BUCKETS + 1)]
            with torch.cuda.device(dev):
                for e in events:                    # torch creates the CUDA event at its first record
                    e.record(side)
            g = _lib.OdometryTrainGroup(rank=r, world=world, multicast=0, n_ctas=n_ctas, n_threads=n_threads,
                                        status=self.status[r].data_ptr(), side_stream=side.cuda_stream,
                                        join_event=events[-1].cuda_event)
            for q in range(world):
                g.peer_ws[q] = workspaces[q].workspace.data_ptr()
                g.peer_flags[q] = self.flags[q].data_ptr()
            for k in range(_lib.TRAIN_GROUP_BUCKETS):
                g.fork_events[k] = events[k].cuda_event
            self.side_streams.append(side)
            self.events.append(events)
            self.groups.append(g)
        for w in workspaces:
            torch.cuda.synchronize(w.workspace.device)

    def step(self, rank, points, counts, outputs=True):
        return self.workspaces[rank].step_group(self.groups[rank], points, counts, outputs)

    def reset_flags(self):
        """Zero every rank's flag words (after a set_state that moved the step count; no step in flight)."""
        for f in self.flags:
            f.zero_()


class AdaptiveStreamsGroupWorkspace(AdaptiveStreamsWorkspace):
    """delora_odometry_streams_adapt_group_*: the adapting-streams layout with the group section appended; every
    AdaptiveStreamsWorkspace call works on it.  `push_group` takes one group tick with a _lib.OdometryTrainGroup."""
    SIZE_QUERY = "delora_odometry_streams_adapt_group_workspace_bytes"

    def _init(self, weights):
        self._call("delora_odometry_streams_adapt_group_init", weights.data_ptr(), self.workspace.data_ptr())

    def push_group(self, group, points, counts, active, T, valid, losses, update=True):
        """AdaptiveStreamsWorkspace.push as rank `group.rank`: with update, the step on the mean over the valid pairs
        of every rank."""
        self._call("delora_odometry_streams_push_adapt_group", self._params, ctypes.byref(group), 1 if update else 0,
                   points.data_ptr(), counts.data_ptr(), _ptr(active), self.workspace.data_ptr(), T.data_ptr(),
                   valid.data_ptr(), losses.data_ptr())


class AdaptingStreamsGroup(TrainingGroup):
    """TrainingGroup over N AdaptiveStreamsGroupWorkspaces (same descriptor and state, N devices with peer access or
    one device): one model adapted from the streams of every rank.  `push(r, ...)` runs rank r's tick on the current
    stream of its device; every rank makes the same number of update = True calls.  Over
    AdaptiveInformationStreamsWorkspaces each tick also returns the information rows."""

    def push(self, rank, points, counts, active, update=True, out=None):
        """points [S, 3, n_stride], counts [S], active [S] int32 or None -> (T [S, 16], valid [S], losses [S, LOSS_ROW])
        and, over information workspaces, info [S, INFO_ROW]; into `out` when given."""
        w = self.workspaces[rank]
        if out is None:
            S, dev = w.desc.max_batch, w.workspace.device
            out = (torch.empty((S, 16), dtype=torch.float32, device=dev), torch.empty((S,), dtype=torch.int32, device=dev),
                   torch.empty((S, ops.LOSS_ROW), dtype=torch.float32, device=dev))
            if isinstance(w, AdaptiveInformationStreamsWorkspace):
                out += (torch.empty((S, ops.INFO_ROW), dtype=torch.float32, device=dev),)
        w.push_group(self.groups[rank], points, counts, active, *out, update=update)
        return out


class AdaptiveInformationStreamsWorkspace(AdaptiveStreamsGroupWorkspace):
    """delora_odometry_streams_adapt_info_*: the group layout of the adapting streams with the information section
    appended; every AdaptiveStreamsWorkspace call works on it.  `push` and `push_group` take info [S, INFO_ROW] out
    after losses: the information row at the served T (before the tick's update) of every valid stream, in the metres
    and radians of T for normalised models too; zeros elsewhere."""
    SIZE_QUERY = "delora_odometry_streams_adapt_info_workspace_bytes"

    def _init(self, weights):
        self._call("delora_odometry_streams_adapt_info_init", weights.data_ptr(), self.workspace.data_ptr())

    def push(self, points, counts, active, T, valid, losses, info, update=True):
        self._call("delora_odometry_streams_push_adapt_info", self._params, 1 if update else 0, points.data_ptr(),
                   counts.data_ptr(), _ptr(active), self.workspace.data_ptr(), T.data_ptr(), valid.data_ptr(),
                   losses.data_ptr(), info.data_ptr())

    def push_group(self, group, points, counts, active, T, valid, losses, info, update=True):
        self._call("delora_odometry_streams_push_adapt_group_info", self._params, ctypes.byref(group),
                   1 if update else 0, points.data_ptr(), counts.data_ptr(), _ptr(active), self.workspace.data_ptr(),
                   T.data_ptr(), valid.data_ptr(), losses.data_ptr(), info.data_ptr())
