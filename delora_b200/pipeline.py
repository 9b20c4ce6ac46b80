"""Batched scan-pair hot path: raw scans -> range images -> normals -> lists -> fused ICP
losses + gradient w.r.t. the predicted transform.  One launch per operator for the whole batch,
all buffers preallocated (no allocation, no host sync inside a step; CUDA-graph capturable).

This is what `Deployer.step` does per sample with Python loops and host round trips
(src/deploy/deployer.py:245-268 projection, :290-312 transform + ICPLosses), with the normals
computed in-line from the projected image as the reference's preprocessing does
(src/preprocessing/preprocesser.py:52,60-61).
"""
import torch

from . import _lib, ops


class ScanPairPipeline:
    def __init__(self, batch, n_max, h, w, hfov, vfov, device="cuda", channels=3, neighborhood=(7, 11),
                 epsilon_range=0.5, min_neighbors=10, lambda_po2pl=1.0,
                 flags=ops.LOSS_PO2PL | ops.LOSS_PL2PL, div_mode=0, concurrency=None):
        self.B, self.N, self.H, self.W, self.C = int(batch), int(n_max), int(h), int(w), int(channels)
        self.hfov, self.vfov = (float(hfov[0]), float(hfov[1])), (float(vfov[0]), float(vfov[1]))
        self.nb, self.eps, self.min_nb = tuple(neighborhood), float(epsilon_range), int(min_neighbors)
        self.lam, self.flags, self.div_mode = float(lambda_po2pl), int(flags), int(div_mode)
        self.device = torch.device(device)
        self.L = _lib.lib()
        if self.device.type != "cuda":
            raise RuntimeError("delora_b200 runs on CUDA devices only (no CPU fallback)")
        b2, hw, dev = 2 * self.B, self.H * self.W, self.device
        f32, i32 = torch.float32, torch.int32
        # the three inputs of a step live in ONE allocation (`inputs`, raw bytes) so that a host caller can ship
        # them with a single pinned-memory copy: [points | n_points | transform], each 256-byte aligned
        self.input_layout = self.staging_layout(self.B, self.C, self.N)
        self.inputs = torch.zeros((self.input_layout["bytes"],), dtype=torch.uint8, device=dev)
        self.points, self.n_points, self.transform = self.input_views(self.inputs, self.input_layout)
        self.keys = torch.full((b2, hw), -1, dtype=torch.int64, device=dev)
        self.image = torch.empty((b2, self.C + 1, self.H, self.W), dtype=f32, device=dev)
        self.index_map = torch.empty((b2, self.H, self.W), dtype=i32, device=dev)
        # dense float4 grids written by the normals kernel: (x,y,z,pixel id) / (nx,ny,nz,has_normal)
        self.pts_grid = torch.empty((b2, hw, 4), dtype=f32, device=dev)
        self.nrm_grid = torch.empty((b2, hw, 4), dtype=f32, device=dev)
        self.losses = torch.empty((self.B, ops.LOSS_ROW), dtype=f32, device=dev)
        self.grad_T = torch.empty((self.B, 12), dtype=f32, device=dev)
        self.icp_scratch = ops.icp_scratch(self.B, hw, dev)       # zeroed once; the kernels keep it armed
        # `concurrency` sub-batches of pairs for the ICP operator, each on its own stream (forked from / joined into the
        # caller's stream inside step()); bit-identical results (every pair is independent).  Default: 2 from 4 pairs up.
        # Projection + normals always run as ONE call for the whole batch on the caller's stream: its normals kernel
        # resolves the projection itself and fills the GPU on its own, so per-sub-batch calls only add launches, wave
        # tails and key re-arms (H100 80GB HBM3 at a 400 W power limit, 8 pairs of 64 x 2048, 4 rotating input sets:
        # ~379 us per step against ~389 us with projection + normals per sub-batch).
        if concurrency is None:
            concurrency = 2 if self.B >= 4 else 1
        self.concurrency = max(1, min(int(concurrency), self.B))
        self._subs = []
        if self.concurrency > 1:
            per = (self.B + self.concurrency - 1) // self.concurrency
            for k in range(self.concurrency):
                b0, b1 = k * per, min(self.B, (k + 1) * per)
                if b1 > b0:
                    self._subs.append({"b0": b0, "n": b1 - b0, "stream": torch.cuda.Stream(device=dev),
                                       "scratch": ops.icp_scratch(b1 - b0, hw, dev), "done": torch.cuda.Event()})
            self._fork = torch.cuda.Event()
        # per step: (scatter + fused resolve / normals + key re-arm memset) + (target_extents + icp_dense +
        # icp_dense_pending + finalize) per ICP sub-batch
        self.launches_per_step = 3 + 4 * max(1, len(self._subs))

    @staticmethod
    def staging_layout(batch, channels, n_max):
        """Byte offsets of (points [2B,C,N] f32, n_points [2B] i32, transform [B,12] f32) inside `inputs`."""
        def up(x):
            return (x + 255) // 256 * 256
        p_bytes = 2 * batch * channels * n_max * 4
        n_off = up(p_bytes)
        t_off = up(n_off + 2 * batch * 4)
        return {"B": batch, "C": channels, "N": n_max, "n_points": n_off, "transform": t_off,
                "bytes": up(t_off + batch * 12 * 4)}

    @staticmethod
    def input_views(buf, layout):
        """Typed views (points, n_points, transform) of a flat uint8 buffer (device `inputs` or a pinned host twin)."""
        b, c, n = layout["B"], layout["C"], layout["N"]
        points = buf[:2 * b * c * n * 4].view(torch.float32).view(2 * b, c, n)       # [scan_1 x B | scan_2 x B]
        n_points = buf[layout["n_points"]:layout["n_points"] + 2 * b * 4].view(torch.int32)
        transform = buf[layout["transform"]:layout["transform"] + b * 48].view(torch.float32).view(b, 12)
        return points, n_points, transform

    def load(self, scans_1, scans_2, transforms):
        """Host-side staging helper for tests: lists of [3,N_i] tensors + [B,4,4] transforms."""
        for i, (s1, s2) in enumerate(zip(scans_1, scans_2)):
            self.points[i, :, :s1.shape[1]] = s1.to(self.device)
            self.points[self.B + i, :, :s2.shape[1]] = s2.to(self.device)
            self.n_points[i] = s1.shape[1]
            self.n_points[self.B + i] = s2.shape[1]
        self.transform.copy_(transforms[:, :3, :].reshape(self.B, 12).to(self.device))

    OPERATORS = ("projection", "normals", "icp")

    def step(self, events=None):
        """Enqueue the whole hot path on the current stream; returns (losses [B,8], grad_T [B,12]).
        `events`: optional list of 4 torch.cuda.Event (timing enabled) recorded before the first and
        after each of the three operators, for per-kernel timing inside a measured region.  Projection and normals
        are one call whose normals kernel also resolves the projection: "projection" ends after its scatter pass."""
        if ops.NVTX:
            torch.cuda.nvtx.range_push("scan-pair step")
            try:
                return self._step(events)
            finally:
                torch.cuda.nvtx.range_pop()
        return self._step(events)

    def _step(self, events):
        if self._subs and events is None:
            return self._step_concurrent()
        L, st = self.L, torch.cuda.current_stream().cuda_stream
        split = None
        if events is not None:
            events[0].record()
            events[1].record()         # creates the event; the call below records it again after the scatter pass
            split = events[1].cuda_event
        b2, B, H, W, hw = 2 * self.B, self.B, self.H, self.W, self.H * self.W
        hf, vf = self.hfov, self.vfov
        _lib.check(L.delora_project_normals_fwd(self.points.data_ptr(), self.n_points.data_ptr(), b2, self.C, self.N,
                                                H, W, hf[0], hf[1], vf[0], vf[1], self.div_mode, self.keys.data_ptr(),
                                                self.image.data_ptr(), self.index_map.data_ptr(), self.nb[0],
                                                self.nb[1], self.eps, self.min_nb, self.pts_grid.data_ptr(),
                                                self.nrm_grid.data_ptr(), split, st), "delora_project_normals_fwd")
        if events is not None:
            events[2].record()
        # source = scan_2 (second half), target = scan_1 (first half): deployer.py:294-307
        f4 = 16
        _lib.check(L.delora_icp_dense_fwd_bwd(self.pts_grid.data_ptr() + B * hw * f4,
                                              self.nrm_grid.data_ptr() + B * hw * f4, self.transform.data_ptr(),
                                              self.pts_grid.data_ptr(), self.nrm_grid.data_ptr(), B, H, W,
                                              hf[0], hf[1], vf[0], vf[1], self.lam, self.flags,
                                              self.losses.data_ptr(), self.grad_T.data_ptr(),
                                              self.icp_scratch.data_ptr(), st), "delora_icp_dense_fwd_bwd")
        if events is not None:
            events[3].record()
        return self.losses, self.grad_T

    def _step_concurrent(self):
        """The same work as step(): projection + normals for the whole batch on the caller's stream, then the ICP as
        `concurrency` independent sub-batches of pairs on their own streams."""
        L, B, H, W, C, N = self.L, self.B, self.H, self.W, self.C, self.N
        hw, hf, vf = H * W, self.hfov, self.vfov
        cur = torch.cuda.current_stream(self.device)
        pts, npt, keys = self.points.data_ptr(), self.n_points.data_ptr(), self.keys.data_ptr()
        img, imap = self.image.data_ptr(), self.index_map.data_ptr()
        pg, ng = self.pts_grid.data_ptr(), self.nrm_grid.data_ptr()
        _lib.check(L.delora_project_normals_fwd(pts, npt, 2 * B, C, N, H, W, hf[0], hf[1], vf[0], vf[1], self.div_mode,
                                                keys, img, imap, self.nb[0], self.nb[1], self.eps, self.min_nb, pg, ng,
                                                None, cur.cuda_stream), "delora_project_normals_fwd")
        self._fork.record(cur)
        for sub in self._subs:
            s, b0, n = sub["stream"], sub["b0"], sub["n"]
            s.wait_event(self._fork)
            st = s.cuda_stream
            _lib.check(L.delora_icp_dense_fwd_bwd(pg + (B + b0) * hw * 16, ng + (B + b0) * hw * 16,
                                                  self.transform.data_ptr() + b0 * 48, pg + b0 * hw * 16,
                                                  ng + b0 * hw * 16, n, H, W, hf[0], hf[1], vf[0], vf[1], self.lam,
                                                  self.flags, self.losses.data_ptr() + b0 * ops.LOSS_ROW * 4,
                                                  self.grad_T.data_ptr() + b0 * 48, sub["scratch"].data_ptr(), st),
                       "delora_icp_dense_fwd_bwd")
            sub["done"].record(s)
            cur.wait_event(sub["done"])
        return self.losses, self.grad_T

    def algorithmic_bytes(self, k_points=None):
        """Algorithmic bytes per launch of each operator (SURVEY.md §8(d) per-unit figures x the units
        one launch processes; DESIGN.md §Measurement).  k_points: mean valid pixels per scan (K)."""
        b2, B, hw, c = 2 * self.B, self.B, self.H * self.W, self.C
        k = float(k_points) if k_points is not None else float(hw)
        n = float(self.N)
        return {
            "projection": b2 * (4 * c * n + 4 * (c + 1) * hw + 4 * hw),          # read xyz, write image + index map
            "normals": b2 * (12 * hw + 12 * hw),                                   # read xyz image, write normals
            "icp": B * ((16 * hw + 12 * k + 4 * k) + (12 * k + 12 * k + 4 * k + 24 * k)),   # NN search + fused loss (K=M)
        }
