"""Streaming odometry inference: the per-frame path of `Tester.test_dataset` / the ROS node
(reference: src/deploy/tester.py:38-107 -> src/deploy/deployer.py:237-281, :370-375;
src/ros_utils/odometry_publisher.py:137-147), one frame at a time, batch 1.

Per frame the reference projects BOTH scans of the pair again (the previous frame's projection is recomputed),
runs the encoder through cuDNN and synchronises with the host three times.  Here a frame costs ONE projection
(the previous frame's range image is kept on the device), the encoder forward on the wgmma kernels and the
quaternion -> T kernel, captured once in a CUDA graph (25 launches replayed as one) between a pinned-memory
H2D of the raw scan and a 64-byte D2H of the relative transform.  BASELINE config #5.

A model trained with normalization_scaling (the ROS node's normalisation, odometry_publisher.py:102-111, :155, :176;
the factor here is the Deployer's, `ops.normalization_factors`) cannot reuse the previous frame's image: it depends on
the factor of the pair.  Such a stream keeps the previous SCAN on the device instead and per frame computes the factor,
divides both scans by it, projects both, runs the model and multiplies the translation back by the factor, again in
one captured graph.

OdometryStreams serves several streams of one sensor geometry and model from one C-ABI workspace, batched; it refuses
normalised models, which NormalizedOdometryStreams serves the same way from the normalised streams workspace.  Both feed
the model raw scans projected at its width (the ROS node's input); PreprocessedOdometryStreams feeds it the images of
the reference's two-resolution recipe (the Tester's and training's input), with an ICP residual per frame.
AdaptiveOdometryStreams serves streams from a training workspace and takes the self-supervised training step on the
pairs it has just served, so the model adapts while it serves.
"""
import numpy as np
import torch

from .. import ops
from ..models import model_parts
from ..utility import poses as poses_module


class OdometryStream:
    def __init__(self, model, config, dataset, n_max, use_cuda_graph=True):
        self.model = model.eval()
        self.config = config
        self.dataset = dataset
        ds = config[dataset]
        self.h, self.w = int(ds["vertical_cells"]), int(ds["horizontal_cells"])
        self.hf, self.vf = config["horizontal_field_of_view"], ds["vertical_field_of_view"]
        self.device = torch.device(config["device"])
        if self.device.type != "cuda":
            raise RuntimeError("OdometryStream runs on CUDA devices only (no CPU fallback)")
        self.n_max = int(n_max)
        self.host_scan = torch.zeros((1, 3, self.n_max), dtype=torch.float32).pin_memory()
        self.host_count = torch.zeros((1,), dtype=torch.int32).pin_memory()
        self.host_T = torch.zeros((1, 4, 4), dtype=torch.float32).pin_memory()
        self._host_scan_np, self._host_count_np = self.host_scan.numpy(), self.host_count.numpy()
        self.normalized = bool(config.get("normalization_scaling", False))
        if self.normalized:
            # rows: the previous scan, this scan; a frame's upload goes to row 1, and row 1 moves to row 0 after it
            self.pair_points = torch.zeros((2, 3, self.n_max), dtype=torch.float32, device=self.device)
            self.pair_counts = torch.zeros((2,), dtype=torch.int32, device=self.device)
            self.points, self.count = self.pair_points[1:], self.pair_counts[1:]
            self.factor = torch.zeros((1,), dtype=torch.float32, device=self.device)
        else:
            self.points = torch.zeros((1, 3, self.n_max), dtype=torch.float32, device=self.device)
            self.count = torch.zeros((1,), dtype=torch.int32, device=self.device)
        self.prev_image = torch.zeros((1, 4, self.h, self.w), dtype=torch.float32, device=self.device)
        self.T = torch.zeros((1, 4, 4), dtype=torch.float32, device=self.device)
        self.frames = 0
        self.relative = []                       # [1,4,4] numpy per frame pair, like Tester's lists
        self.use_cuda_graph = bool(use_cuda_graph)
        self.graph = None
        # the model's own configuration decides the encoder path (tensor cores by default when eligible,
        # models/model.py); the stream never edits the shared config dict

    # everything of a frame that runs on the device; static shapes and buffers (graph-capturable)
    def _frame(self):
        if self.normalized:
            return self._frame_normalized()
        image, _ = ops.project(self.points, self.count, self.h, self.w, self.hf, self.vf)     # closest point per pixel
        with torch.no_grad():
            translation, quaternion = self.model(image_1=self.prev_image, image_2=image)
            t = model_parts.GeometryHandler.get_transformation_matrix_quaternion(
                translation=translation, quaternion=quaternion, device=self.device)
        self.T.copy_(t)
        self.prev_image.copy_(image)

    def _frame_normalized(self):
        factor = ops.normalization_factors(self.pair_points, self.pair_counts)                # [1]
        scaled = self.pair_points / factor.view(1, 1, 1)
        image, _ = ops.project(scaled, self.pair_counts, self.h, self.w, self.hf, self.vf)
        self.pair_image = image                  # [previous, this] as the model saw them (the graph's output under replay)
        with torch.no_grad():
            translation, quaternion = self.model(image_1=image[0:1], image_2=image[1:2])
            t = model_parts.GeometryHandler.get_transformation_matrix_quaternion(
                translation=translation, quaternion=quaternion, device=self.device)
        t[:, :3, 3] *= factor.view(1, 1)
        self.T.copy_(t)
        self.factor.copy_(factor)
        self._advance()

    def _advance(self):
        """Normalised route: this scan becomes the previous one."""
        self.pair_points[0].copy_(self.pair_points[1])
        self.pair_counts[0].copy_(self.pair_counts[1])

    def _capture(self):
        if self.normalized:
            return self._capture_normalized()
        side = torch.cuda.Stream(device=self.device)
        saved = self.prev_image.clone()          # taken BEFORE the side stream is released: the warm-up frames write prev_image
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):                   # warm-up: allocator, tensor-map cache, cuBLAS handles
                self._frame()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._frame()
        self.prev_image.copy_(saved)

    def _capture_normalized(self):
        # the warm-up frames overwrite the previous scan with this one: restore it before the first replay
        saved = (self.pair_points[0].clone(), self.pair_counts[0].clone())
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                self._frame()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self._frame()
        self.pair_points[0].copy_(saved[0])
        self.pair_counts[0].copy_(saved[1])

    def push(self, scan):
        """scan: [3,N] or [1,3,N] float32 host tensor (N <= n_max).  Returns the relative transform
        T_{k-1,k} as a [1,4,4] numpy array, or None for the first frame of a stream."""
        scan = scan[0] if scan.dim() == 3 else scan
        n = int(scan.shape[1])
        if n > self.n_max:
            raise Exception("scan has more points than the stream was sized for")
        # plain memcpy into the pinned staging buffer: a torch copy of this size wakes the intra-op thread pool, whose
        # spinning workers can exhaust a container's CPU quota and stall the stream for tens of ms every 100 ms
        np.copyto(self._host_scan_np[0, :, :n], scan[:3].numpy())
        self._host_count_np[0] = n
        self.points.copy_(self.host_scan, non_blocking=True)
        self.count.copy_(self.host_count, non_blocking=True)
        first = self.frames == 0
        if first:
            # no previous frame yet: project only (normalised route: keep the scan)
            if self.normalized:
                self._advance()
            else:
                image, _ = ops.project(self.points, self.count, self.h, self.w, self.hf, self.vf)
                self.prev_image.copy_(image)
            torch.cuda.current_stream().synchronize()
            self.frames += 1
            return None
        tc = self.model._tensor_core_path()
        if tc is not None:
            tc._refresh_weights()                # bf16 filter copies follow the fp32 parameters (no-op when unchanged)
        if self.use_cuda_graph:
            if self.graph is None:
                self._capture()
            self.graph.replay()
        else:
            self._frame()
        self.host_T.copy_(self.T, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.frames += 1
        t = self.host_T.numpy().copy()
        self.relative.append(t)
        return t

    def poses(self):
        """World-frame KITTI poses of the stream so far (src/utility/poses.py:11-58)."""
        return poses_module.compute_poses(self.relative)

    def reset(self):
        self.frames = 0
        self.relative = []


def _staging(fields, device):
    """One pinned host buffer and one device buffer holding the 4-byte fields [(name, shape, dtype), ...] back to back.
    Returns both buffers, the host views by name and the device slices in field order."""
    sizes = [4 * int(np.prod(shape)) for _, shape, _ in fields]
    host = torch.zeros((sum(sizes),), dtype=torch.uint8).pin_memory()
    dev = torch.zeros((sum(sizes),), dtype=torch.uint8, device=device)
    raw, views, slices, off = host.numpy(), {}, [], 0
    for (name, shape, dtype), size in zip(fields, sizes):
        views[name] = raw[off:off + size].view(dtype).reshape(shape)
        slices.append(dev[off:off + size])
        off += size
    return host, dev, views, slices


class _Streams:
    """What the streams front-ends share: the host fill of a tick's scans, the per-stream results, poses and reset.
    A subclass sets n_streams, n_max, device, workspace, relative (one list per stream) and _mask (device int32 [S])."""

    def _fill(self, scans, points, counts, active):
        """scans (see push) into the host arrays points [S, 3, n_max], counts [S] and active [S]."""
        if len(scans) != self.n_streams:
            raise ValueError(f"push takes {self.n_streams} entries (one per stream, None = inactive), got {len(scans)}")
        for s, scan in enumerate(scans):
            if scan is None:
                active[s] = 0
                counts[s] = 0
                continue
            scan = scan[0] if scan.dim() == 3 else scan
            n = int(scan.shape[1])
            if n > self.n_max:
                raise ValueError(f"stream {s}: scan has more points than the streams were sized for")
            np.copyto(points[s, :, :n], scan[:3].numpy())
            counts[s] = n
            active[s] = 1

    def _results(self, T, valid, extras):
        """Per stream: None without a transform; else T [1, 4, 4] (kept for poses), or with extras (arrays with a row
        per stream) the tuple (T, row of each extra), a 1-D extra's row as a float."""
        out = []
        for s in range(self.n_streams):
            if not valid[s]:
                out.append(None)
                continue
            t = T[s].reshape(1, 4, 4).copy()
            self.relative[s].append(t)
            rows = tuple(e[s].copy() if e.ndim > 1 else float(e[s]) for e in extras)
            out.append((t,) + rows if extras else t)
        return out

    def poses(self, s):
        """World-frame KITTI poses of stream s so far (src/utility/poses.py:11-58)."""
        return poses_module.compute_poses(self.relative[s])

    def reset(self, s):
        """Forget stream s's previous frame and its transforms: its next frame starts it again."""
        with torch.cuda.device(self.device):
            self._mask.zero_()
            self._mask[s] = 1
            self.workspace.reset(self._mask)
            torch.cuda.current_stream().synchronize()
        self.relative[s] = []


class OdometryStreams(_Streams):
    """Several LiDAR streams (sensors of one robot, or vehicles served by one process) through one streams workspace of
    the C ABI (`delora_odometry_streams_*`): all streams share the image geometry and the model, and one tick runs the
    model once at batch `n_streams`.  Each stream's transforms are bit-identical to a `delora_odometry_push` workspace
    fed only that stream's frames (each quaternion is divided by its own row's norm, as at batch 1).

    Per tick: the scans are copied into one pinned staging buffer (points, counts, activity flags), one H2D copy, one
    graph replay (or the eager call), one D2H copy of T and valid, one synchronise.

    residual=True serves the streams from the residual workspace (`delora_odometry_streams_push_residual`): `push` then
    returns, beside each transform, the stream's ICP loss row [LOSS_ROW] (po2po, po2pl, pl2pl, matched pairs, matched
    po2po pairs, ...) of this frame moved by T against the previous frame, with the normals estimated on the model's
    H x W image and the config's neighbourhood; `residual_flags` selects the losses (None: the objective the config
    names, po2po_alone included, as a .dlw records it).  The transforms are the same bits either way."""

    def __init__(self, model, config, dataset, n_streams, n_max, use_cuda_graph=True, residual=False,
                 residual_flags=None):
        if config.get("normalization_scaling", False):
            raise ValueError("normalization_scaling: True is not supported by OdometryStreams (its workspace caches "
                             "each stream's projected image, which a normalised model cannot reuse); serve such a "
                             "model with NormalizedOdometryStreams")
        self._setup(model, config, dataset, n_streams, n_max, use_cuda_graph, residual, residual_flags, False)

    def _setup(self, model, config, dataset, n_streams, n_max, use_cuda_graph, residual, residual_flags, normalized,
               pre=False, info=False):
        from . import capi, export
        self.config = config
        self.dataset = dataset
        self.device = torch.device(config["device"])
        if self.device.type != "cuda":
            raise RuntimeError("OdometryStreams runs on CUDA devices only (no CPU fallback)")
        self.n_streams, self.n_max = int(n_streams), int(n_max)
        self.desc = export.desc_from_config(config, dataset, self.n_max, self.n_streams, preprocessing_normals=pre)
        S, n = self.n_streams, self.n_max
        self.residual = bool(residual) or pre
        self.normalized = bool(normalized)
        # the tick's outputs in the order the workspace's push takes them: T and valid, the residual's losses, the
        # information rows, the normalised kinds' factor
        outputs = [("T", (S, 4, 4), np.float32), ("valid", (S,), np.int32)]
        if self.residual:
            outputs.append(("losses", (S, ops.LOSS_ROW), np.float32))
        if info:
            outputs.append(("info", (S, ops.INFO_ROW), np.float32))
        if normalized:
            outputs.append(("factor", (S,), np.float32))
        with torch.cuda.device(self.device):
            self.blob = torch.from_numpy(export.pack_state_dict(model.state_dict(), config)).to(self.device)
            if pre:
                if residual_flags is None:
                    residual_flags = export.objective_from_config(config)[0]
                flags = residual_flags | (ops.TRAIN_NORMALIZATION_SCALING if normalized else 0)
                kind = capi.PreInformationStreamsWorkspace if info else capi.PreStreamsWorkspace
                self.workspace = kind(self.desc, self.blob, capi.residual_params(config, flags))
            elif info:
                self.workspace = capi.InformationStreamsWorkspace(self.desc, self.blob,
                                                                  capi.residual_params(config, residual_flags))
            elif self.residual:
                self.workspace = capi.ResidualStreamsWorkspace(self.desc, self.blob,
                                                               capi.residual_params(config, residual_flags))
            elif normalized:
                self.workspace = capi.NormalizedStreamsWorkspace(self.desc, self.blob)
            else:
                self.workspace = capi.StreamsWorkspace(self.desc, self.blob)
            self.host_in, self.dev_in, self._in, dev_in = _staging(
                [("points", (S, 3, n), np.float32), ("counts", (S,), np.int32), ("active", (S,), np.int32)],
                self.device)
            self.host_out, self.dev_out, self._out, dev_out = _staging(outputs, self.device)
            self._mask = torch.zeros((S,), dtype=torch.int32, device=self.device)
        # the push arguments of a tick, all in the device staging buffers
        self._dev_active = dev_in[2]
        self._tick = tuple(dev_in) + tuple(dev_out)
        # what push returns beside T: the residual's losses, the information rows and the recipe's factor (the
        # normalised raw-scan streams return T alone)
        self._extras = (([self._out["losses"]] if self.residual else []) + ([self._out["info"]] if info else []) +
                        ([self._out["factor"]] if pre and normalized else []))
        self.relative = [[] for _ in range(S)]
        self.use_cuda_graph = bool(use_cuda_graph)
        self.graph = None

    def _capture(self):
        # a tick with every stream inactive changes no stream's state: it warms the launchers' host-side caches, then
        # the call is captured (capturing runs nothing)
        torch.cuda.current_stream().synchronize()
        self._dev_active.zero_()
        self.workspace.push(*self._tick)
        torch.cuda.current_stream().synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.workspace.push(*self._tick)

    def push(self, scans):
        """scans: a list of n_streams entries, each a [3, N] (or [1, 3, N]) float32 host tensor with N <= n_max, or
        None for a stream without a frame this tick.  Returns a list of n_streams entries: the relative transform
        T_{k-1,k} of the stream as a [1, 4, 4] numpy array, or None (no frame, or the stream's first frame).  With
        residual=True an entry with a transform is the tuple (T, losses [LOSS_ROW] numpy array)."""
        self._fill(scans, self._in["points"], self._in["counts"], self._in["active"])
        with torch.cuda.device(self.device):
            if self.use_cuda_graph and self.graph is None:
                self._capture()
            self.dev_in.copy_(self.host_in, non_blocking=True)
            if self.graph is not None:
                self.graph.replay()
            else:
                self.workspace.push(*self._tick)
            self.host_out.copy_(self.dev_out, non_blocking=True)
            torch.cuda.current_stream().synchronize()
        return self._results(self._out["T"], self._out["valid"], self._extras)


class InformationOdometryStreams(OdometryStreams):
    """OdometryStreams served from the information workspace (`delora_odometry_streams_push_info`): `push` returns, per
    stream with a transform, (T [1, 4, 4], losses [LOSS_ROW], info [INFO_ROW]).  losses is residual=True's row; info
    is the Gauss-Newton information of that residual's objective at T (include/delora_b200.h, DELORA_INFO_ROW): H
    [0:36] (6 x 6, xi = (x, y, z, rot x, rot y, rot z) perturbing T on the right), its eigenvalues ascending [36:42]
    and their unit eigenvectors [42:78], M and M' [78:80].  A small eigenvalue is a direction of the pose the frame
    does not determine (a corridor, an open field, a flat wall).  The transforms and losses are the same bits as
    residual=True's; `residual_flags` selects the losses; `poses` and `reset` are OdometryStreams'."""

    def __init__(self, model, config, dataset, n_streams, n_max, use_cuda_graph=True,
                 residual_flags=None):
        if config.get("normalization_scaling", False):
            raise ValueError("normalization_scaling: True is not supported by InformationOdometryStreams (the "
                             "information is that of the residual workspace, which serves plain models)")
        self._setup(model, config, dataset, n_streams, n_max, use_cuda_graph, True, residual_flags, False, info=True)


class NormalizedOdometryStreams(OdometryStreams):
    """OdometryStreams for a model trained with normalization_scaling, through the normalised streams workspace
    (`delora_odometry_streams_push_normalized`): the workspace keeps each stream's previous scan, and one tick divides
    both scans of every pair by that pair's factor, projects them, runs the model once at batch `n_streams` and
    multiplies each translation back by its factor.  Each stream's transforms are bit-identical to
    `delora_odometry_pairs_normalized` at batch 1 on (its previous frame, this frame).  Same constructor (without the
    residual), `push`, `poses` and `reset` as OdometryStreams."""

    def __init__(self, model, config, dataset, n_streams, n_max, use_cuda_graph=True):
        if not config.get("normalization_scaling", False):
            raise ValueError("NormalizedOdometryStreams serves models trained with normalization_scaling: True; this "
                             "config has normalization_scaling off, so serve it with OdometryStreams")
        self._setup(model, config, dataset, n_streams, n_max, use_cuda_graph, False, None, True)


class PreprocessedOdometryStreams(OdometryStreams):
    """OdometryStreams on the reference's two-resolution recipe, through the recipe streams workspace
    (`delora_odometry_streams_push_pre`): each frame is projected with its normals at `horizontal_cells_preprocessing`
    (w_pre) and those points are projected again at the model's width, the images a model trained with
    `--preprocessing-normals` saw in training and the reference's Tester feeds it.  Serves plain and
    normalization_scaling configs alike.  `push` returns, per stream with a transform, (T [1, 4, 4], losses [LOSS_ROW])
    -- the training step's ICP residual of the pair, in the model's units -- plus the pair's factor for a normalised
    config: (T, losses, factor).  `residual_flags` selects the losses; `poses` and `reset` are OdometryStreams'.

    information=True serves them from the recipe information workspace (`delora_odometry_streams_push_pre_info`):
    each entry is then (T, losses, info [INFO_ROW][, factor]), info being the Gauss-Newton information of the residual's
    objective at T (see InformationOdometryStreams), in the metres and radians of T for normalised configs too.  T,
    losses and factor are the same bits either way."""

    def __init__(self, model, config, dataset, n_streams, n_max, use_cuda_graph=True,
                 residual_flags=None, information=False):
        if "horizontal_cells_preprocessing" not in config[dataset]:
            raise ValueError(f"{dataset}: horizontal_cells_preprocessing is missing; PreprocessedOdometryStreams "
                             "serves the recipe's normals at that width (serve raw scans with OdometryStreams)")
        self._setup(model, config, dataset, n_streams, n_max, use_cuda_graph, True, residual_flags,
                    bool(config.get("normalization_scaling", False)), pre=True, info=bool(information))


class AdaptiveOdometryStreams(_Streams):
    """Several streams served while the model adapts to them (`delora_odometry_streams_push_adapt`): one tick runs the
    training step's forward at batch `n_streams`, each pair's first frame taken from the workspace, returns each
    stream's T and ICP loss row, and with update=True takes one Adam step (learning rate `lr`, torch's default betas)
    on the mean objective of the pairs it served (`loss_flags`, or None for the objective the config names, po2po_alone
    included).  T is always that of the weights before the tick's update; the next tick serves the updated model.  Normals at the model's width, or with preprocessing_normals=True at
    `horizontal_cells_preprocessing` (the reference's recipe, which normalization_scaling needs).  `state_dict()` is the
    adapted model.  Dropout configs are refused: the served T must be dropout-free.

    information=True serves them from the adapting information workspace (`delora_odometry_streams_push_adapt_info`):
    each entry is then (T, losses, info [INFO_ROW]), info being the Gauss-Newton information of the tick's ICP objective
    at the served T (see InformationOdometryStreams), in the metres and radians of T for normalised configs too.  T,
    losses and the adapted model are the same bits either way."""

    information = False

    def __init__(self, model, config, dataset, n_streams, n_max, lr, preprocessing_normals=False,
                 loss_flags=None, information=False):
        from . import capi, export
        if config.get("use_dropout", False):
            raise ValueError("use_dropout: True is not supported by AdaptiveOdometryStreams: the served transforms "
                             "are dropout-free, and one forward cannot be both")
        if config.get("normalization_scaling", False) and not preprocessing_normals:
            raise ValueError("normalization_scaling: True needs preprocessing_normals=True (the reference's recipe: "
                             "normals from the unscaled points at horizontal_cells_preprocessing)")
        self.config = config
        self.device = torch.device(config["device"])
        if self.device.type != "cuda":
            raise RuntimeError("AdaptiveOdometryStreams runs on CUDA devices only (no CPU fallback)")
        self.n_streams, self.n_max = int(n_streams), int(n_max)
        self.desc = export.desc_from_config(config, dataset, self.n_max, self.n_streams,
                                            preprocessing_normals=preprocessing_normals)
        self.information = bool(information)
        with torch.cuda.device(self.device):
            blob = torch.from_numpy(export.pack_state_dict(model.state_dict(), config)).to(self.device)
            kind = capi.AdaptiveInformationStreamsWorkspace if self.information else capi.AdaptiveStreamsWorkspace
            self.workspace = kind(self.desc, blob, capi.train_params(config, lr, loss_flags=loss_flags))
        self._buffers()

    def _buffers(self):
        S, n = self.n_streams, self.n_max
        with torch.cuda.device(self.device):
            self.points = torch.zeros((S, 3, n), dtype=torch.float32, device=self.device)
            self.counts = torch.zeros((S,), dtype=torch.int32, device=self.device)
            self.active = torch.zeros((S,), dtype=torch.int32, device=self.device)
            self.T = torch.zeros((S, 16), dtype=torch.float32, device=self.device)
            self.valid = torch.zeros((S,), dtype=torch.int32, device=self.device)
            self.losses = torch.zeros((S, ops.LOSS_ROW), dtype=torch.float32, device=self.device)
            self.info = torch.zeros((S, ops.INFO_ROW), dtype=torch.float32, device=self.device)
            self._mask = torch.zeros((S,), dtype=torch.int32, device=self.device)
        self.relative = [[] for _ in range(S)]

    def push(self, scans, update=True):
        """scans: n_streams entries, each a [3, N] (or [1, 3, N]) float32 host tensor with N <= n_max, or None.  Returns
        n_streams entries: (T [1, 4, 4], losses [LOSS_ROW]) numpy arrays for a stream with a pair this tick, else None;
        with information=True, (T, losses, info [INFO_ROW])."""
        pts = torch.zeros((self.n_streams, 3, self.n_max), dtype=torch.float32)
        counts = torch.zeros((self.n_streams,), dtype=torch.int32)
        active = torch.zeros((self.n_streams,), dtype=torch.int32)
        self._fill(scans, pts.numpy(), counts.numpy(), active.numpy())
        with torch.cuda.device(self.device):
            self.points.copy_(pts)
            self.counts.copy_(counts)
            self.active.copy_(active)
            self._push_device(update)
            T, valid, losses = self.T.cpu().numpy(), self.valid.cpu().numpy(), self.losses.cpu().numpy()
            extras = [losses, self.info.cpu().numpy()] if self.information else [losses]
        return self._results(T, valid, extras)

    def _push_device(self, update):
        if self.information:
            self.workspace.push(self.points, self.counts, self.active, self.T, self.valid, self.losses, self.info, update)
        else:
            self.workspace.push(self.points, self.counts, self.active, self.T, self.valid, self.losses, update)

    def state_dict(self):
        """The adapted weights as an OdometryModel state dict (fp32 CPU tensors)."""
        from . import export
        with torch.cuda.device(self.device):
            w = self.workspace.weights().cpu().numpy()
        return export.unpack_blob(w, self.config)


class GeometriesAdaptiveOdometryStreams(AdaptiveOdometryStreams):
    """AdaptiveOdometryStreams over streams of several sensor geometries in one workspace
    (`delora_odometry_streams_push_adapt_geometries`): `geometries` lists (dataset, n_streams) pairs, each dataset a
    section of `config` with its own image size, vertical field of view and preprocessing width; streams are numbered
    in that order.  One tick serves every geometry's streams, and with update=True takes one Adam step on the mean
    objective over the pairs of all of them, so one model adapts to the whole fleet.  The datasets must share the
    parity of their horizontal_cells.  `push`, `poses`, `reset` and `state_dict` are AdaptiveOdometryStreams'.

    information=True serves them from the geometries information workspace
    (`delora_odometry_streams_push_adapt_geometries_info`): each entry is then (T, losses, info [INFO_ROW]), as for
    AdaptiveOdometryStreams(information=True).  T, losses and the adapted model are the same bits either way."""

    def __init__(self, model, config, geometries, n_max, lr, preprocessing_normals=False,
                 loss_flags=None, information=False):
        from . import capi, export
        if config.get("use_dropout", False):
            raise ValueError("use_dropout: True is not supported by GeometriesAdaptiveOdometryStreams: the served "
                             "transforms are dropout-free, and one forward cannot be both")
        if config.get("normalization_scaling", False) and not preprocessing_normals:
            raise ValueError("normalization_scaling: True needs preprocessing_normals=True (the reference's recipe: "
                             "normals from the unscaled points at horizontal_cells_preprocessing)")
        self.config = config
        self.device = torch.device(config["device"])
        if self.device.type != "cuda":
            raise RuntimeError("GeometriesAdaptiveOdometryStreams runs on CUDA devices only (no CPU fallback)")
        self.n_max = int(n_max)
        self.descs = [export.desc_from_config(config, ds, self.n_max, int(s), preprocessing_normals=preprocessing_normals)
                      for ds, s in geometries]
        self.rows = np.cumsum([0] + [int(s) for _, s in geometries]).tolist()
        self.n_streams = self.rows[-1]
        self.information = bool(information)
        with torch.cuda.device(self.device):
            blob = torch.from_numpy(export.pack_state_dict(model.state_dict(), config)).to(self.device)
            kind = (capi.GeometriesAdaptingInformationStreamsWorkspace if self.information
                    else capi.GeometriesAdaptingStreamsWorkspace)
            self.workspace = kind(self.descs, blob, capi.train_params(config, lr, loss_flags=loss_flags))
        self._buffers()

    def _push_device(self, update):
        r = self.rows
        pts = [self.points[r[g]:r[g + 1]] for g in range(len(self.descs))]
        counts = [self.counts[r[g]:r[g + 1]] for g in range(len(self.descs))]
        extras = (self.info,) if self.information else ()
        self.workspace.push(pts, counts, self.active, self.T, self.valid, self.losses, *extras, update=update)
