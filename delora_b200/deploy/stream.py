"""Streaming odometry inference: the per-frame path of `Tester.test_dataset` / the ROS node
(reference: src/deploy/tester.py:38-107 -> src/deploy/deployer.py:237-281, :370-375;
src/ros_utils/odometry_publisher.py:137-147), one frame at a time, batch 1.

Per frame the reference projects BOTH scans of the pair again (the previous frame's projection is recomputed),
runs the encoder through cuDNN and synchronises with the host three times.  Here a frame costs ONE projection
(the previous frame's range image is kept on the device), the encoder forward on the wgmma kernels and the
quaternion -> T kernel, captured once in a CUDA graph (25 launches replayed as one) between a pinned-memory
H2D of the raw scan and a 64-byte D2H of the relative transform.  BASELINE config #5.

OdometryStreams serves several streams of one sensor geometry and model from one C-ABI workspace, batched.
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
        image, _ = ops.project(self.points, self.count, self.h, self.w, self.hf, self.vf)     # closest point per pixel
        with torch.no_grad():
            translation, quaternion = self.model(image_1=self.prev_image, image_2=image)
            t = model_parts.GeometryHandler.get_transformation_matrix_quaternion(
                translation=translation, quaternion=quaternion, device=self.device)
        self.T.copy_(t)
        self.prev_image.copy_(image)

    def _capture(self):
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
            # no previous frame yet: project only
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


class OdometryStreams:
    """Several LiDAR streams (sensors of one robot, or vehicles served by one process) through one streams workspace of
    the C ABI (`delora_odometry_streams_*`): all streams share the image geometry and the model, and one tick runs the
    model once at batch `n_streams`.  Each stream's transforms are bit-identical to a `delora_odometry_push` workspace
    fed only that stream's frames (each quaternion is divided by its own row's norm, as at batch 1).

    Per tick: the scans are copied into one pinned staging buffer (points, counts, activity flags), one H2D copy, one
    graph replay (or the eager call), one D2H copy of T and valid, one synchronise."""

    def __init__(self, model, config, dataset, n_streams, n_max, use_cuda_graph=True):
        from . import capi, export
        self.config = config
        self.dataset = dataset
        self.device = torch.device(config["device"])
        if self.device.type != "cuda":
            raise RuntimeError("OdometryStreams runs on CUDA devices only (no CPU fallback)")
        self.n_streams, self.n_max = int(n_streams), int(n_max)
        self.desc = export.desc_from_config(config, dataset, self.n_max, self.n_streams)
        S, n = self.n_streams, self.n_max
        with torch.cuda.device(self.device):
            self.blob = torch.from_numpy(export.pack_state_dict(model.state_dict(), config)).to(self.device)
            self.workspace = capi.StreamsWorkspace(self.desc, self.blob)
            # staging: points [S, 3, n_max] fp32, then counts [S] and active [S] int32, one buffer each way
            in_bytes = S * 3 * n * 4 + 2 * S * 4
            self.host_in = torch.zeros((in_bytes,), dtype=torch.uint8).pin_memory()
            self.dev_in = torch.zeros((in_bytes,), dtype=torch.uint8, device=self.device)
            out_bytes = S * 16 * 4 + S * 4                       # T [S, 16] fp32, valid [S] int32
            self.host_out = torch.zeros((out_bytes,), dtype=torch.uint8).pin_memory()
            self.dev_out = torch.zeros((out_bytes,), dtype=torch.uint8, device=self.device)
            self.dev_mask = torch.zeros((S,), dtype=torch.int32, device=self.device)
        raw = self.host_in.numpy()
        self._host_points = raw[:S * 3 * n * 4].view(np.float32).reshape(S, 3, n)
        self._host_counts = raw[S * 3 * n * 4:S * 3 * n * 4 + S * 4].view(np.int32)
        self._host_active = raw[S * 3 * n * 4 + S * 4:].view(np.int32)
        out = self.host_out.numpy()
        self._host_T = out[:S * 64].view(np.float32).reshape(S, 4, 4)
        self._host_valid = out[S * 64:].view(np.int32)
        # the push arguments of a tick: points, counts, active, T, valid in the device staging buffers
        self._dev_active = self.dev_in[S * 3 * n * 4 + S * 4:]
        self._tick = (self.dev_in[:S * 3 * n * 4], self.dev_in[S * 3 * n * 4:S * 3 * n * 4 + S * 4], self._dev_active,
                      self.dev_out[:S * 64], self.dev_out[S * 64:])
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
        T_{k-1,k} of the stream as a [1, 4, 4] numpy array, or None (no frame, or the stream's first frame)."""
        if len(scans) != self.n_streams:
            raise ValueError(f"push takes {self.n_streams} entries (one per stream, None = inactive), got {len(scans)}")
        with torch.cuda.device(self.device):
            if self.use_cuda_graph and self.graph is None:
                self._capture()
            for s, scan in enumerate(scans):
                if scan is None:
                    self._host_active[s] = 0
                    self._host_counts[s] = 0
                    continue
                scan = scan[0] if scan.dim() == 3 else scan
                n = int(scan.shape[1])
                if n > self.n_max:
                    raise Exception(f"stream {s}: scan has more points than the streams were sized for")
                np.copyto(self._host_points[s, :, :n], scan[:3].numpy())
                self._host_counts[s] = n
                self._host_active[s] = 1
            self.dev_in.copy_(self.host_in, non_blocking=True)
            if self.graph is not None:
                self.graph.replay()
            else:
                self.workspace.push(*self._tick)
            self.host_out.copy_(self.dev_out, non_blocking=True)
            torch.cuda.current_stream().synchronize()
        out = []
        for s in range(self.n_streams):
            if self._host_valid[s]:
                t = self._host_T[s][None].copy()
                self.relative[s].append(t)
                out.append(t)
            else:
                out.append(None)
        return out

    def poses(self, s):
        """World-frame KITTI poses of stream s so far (src/utility/poses.py:11-58)."""
        return poses_module.compute_poses(self.relative[s])

    def reset(self, s):
        """Forget stream s's previous frame and its transforms: its next frame starts it again."""
        with torch.cuda.device(self.device):
            self.dev_mask.zero_()
            self.dev_mask[s] = 1
            self.workspace.reset(self.dev_mask)
            torch.cuda.current_stream().synchronize()
        self.relative[s] = []
