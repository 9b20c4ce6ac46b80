"""Shared inputs and Python reference steps of the odometry C-ABI tests (test infrastructure, imported like helpers).

Every input is seeded: the scans by their pair index, the models by `seed`.  The scan tuples are cached and shared by
every module that asks for the same ones, so no caller may modify them in place."""
import collections
import copy
import functools
import os
import subprocess

import numpy as np
import torch

from delora_b200 import ops
from helpers import ROOT

DEV = "cuda:0"
VFOV = (-24.5, 2.0)
FLAGS = ops.LOSS_PO2PL | ops.LOSS_PL2PL          # SyntheticTrainStep's losses
# Gradient bounds of the C training step against the Python step, relative to each tensor's max-abs (the reasoning is
# in test_gpu_odometry_train_capi.py's docstring): the fc / head tensors, and the trunk's
TAIL_TOL = 5e-6
TRUNK_TOL = 1e-2


def config(h, w, act="tanh", single=False, layers=(2, 2, 2, 2), nout=1000, vfov=VFOV, device=DEV):
    from delora_b200 import synthetic
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vfov, device=device)
    cfg.update({"activation_fct": act, "use_single_mlp_at_output": single, "layers": list(layers), "resnet_outputs": nout,
                "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1, "use_dropout": False})
    return cfg


def model(cfg, seed=0, near_identity=False):
    """OdometryModel on DEV with torch's initialisation (train mode) after torch.manual_seed(seed).  near_identity:
    small last layers and the identity quaternion as bias, so T is near I (as after the reference's identity
    pre-training) and every layer gets a gradient."""
    from delora_b200.models.model import OdometryModel
    torch.manual_seed(seed)
    m = OdometryModel(cfg).to(DEV)
    if not near_identity:
        return m
    with torch.no_grad():
        if cfg["use_single_mlp_at_output"]:
            last = m.fully_connected_rot_trans[-1]
            last.weight.mul_(0.01)
            last.bias.copy_(torch.tensor([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]))
        else:
            for head, bias in ((m.fully_connected_rotation, [0.0, 0.0, 0.0, 1.0]),
                               (m.fully_connected_translation, [0.0, 0.0, 0.0])):
                head[3].weight.mul_(0.01)
                head[3].bias.copy_(torch.tensor(bias))
    return m


@functools.lru_cache(maxsize=None)
def pairs(rings, w_raw, count):
    """(scan_1, scan_2) of synthetic pairs 0 .. count-1."""
    from delora_b200 import synthetic
    return tuple(synthetic.make_pair(i, w_raw=w_raw, rings=rings, vfov_deg=VFOV)[:2] for i in range(count))


def frames(rings, w_raw, count):
    """Consecutive synthetic frames: scan_1, scan_2 of pair 0, scan_1, scan_2 of pair 1, ..."""
    return tuple(s for p in pairs(rings, w_raw, (count + 1) // 2) for s in p)[:count]


def n_stride(pair_list):
    return max(max(a.shape[1], b.shape[1]) for a, b in pair_list)


def stack(scans, stride):
    """Scans -> points [len, 3, n_stride] (zero padded) and counts [len] on DEV."""
    pts = torch.zeros((len(scans), 3, stride), dtype=torch.float32)
    for i, s in enumerate(scans):
        pts[i, :, :s.shape[1]] = s
    counts = torch.tensor([s.shape[1] for s in scans], dtype=torch.int32)
    return pts.to(DEV), counts.to(DEV)


def stack_pairs(pair_list, stride):
    """The rows of a step on these pairs: scan_1 x B, then scan_2 x B."""
    return stack([p[0] for p in pair_list] + [p[1] for p in pair_list], stride)


def blob(m, cfg):
    from delora_b200.deploy import export
    return torch.from_numpy(export.pack_state_dict(m.state_dict(), cfg)).to(DEV)


def desc(cfg, stride, max_batch, w_pre=0):
    from delora_b200.deploy import export
    d = export.desc_from_config(cfg, "kitti", stride, max_batch)
    d.w_pre = w_pre
    return d


def trainer(cfg, stride, max_batch, weights, lr=1e-5, w_pre=0, flags=FLAGS):
    from delora_b200.deploy import capi
    return capi.TrainingWorkspace(desc(cfg, stride, max_batch, w_pre), weights,
                                  capi.train_params(cfg, lr, loss_flags=flags))


def _preprocessed_lists(cfg, pts, counts, w_pre):
    """The offline stage (Preprocesser.preprocess_scans at horizontal_cells_preprocessing = w_pre) of every scan ->
    padded channels-first point and normal lists [2B, 3, P] and their lengths [2B]."""
    from delora_b200.preprocessing.normal_computation import NormalsComputer
    from delora_b200.preprocessing.preprocesser import Preprocesser
    pcfg = copy.deepcopy(cfg)
    pcfg["dataset"] = "kitti"
    pcfg["kitti"]["horizontal_cells"] = w_pre
    pre = Preprocesser(config=pcfg)
    pre.normals_computer = NormalsComputer(config=pcfg, dataset_name="kitti")
    n_host = counts.cpu().tolist()
    out = pre.preprocess_scans([pts[i, :, :n].cpu() for i, n in enumerate(n_host)])
    p_max = max(max(p.shape[0] for _, p in out), 1)
    plist = torch.zeros((len(out), 3, p_max), dtype=torch.float32)
    nlist = torch.zeros_like(plist)
    for i, (nrm, p) in enumerate(out):
        plist[i, :, :p.shape[0]] = torch.from_numpy(p).t()
        nlist[i, :, :nrm.shape[0]] = torch.from_numpy(nrm).t()
    lens = torch.tensor([p.shape[0] for _, p in out], dtype=torch.int32)
    return plist.to(DEV), nlist.to(DEV), lens.to(DEV)


Step = collections.namedtuple("Step", "losses T pooled grads objective")


def python_step(m, cfg, pts, counts, w_pre=0, identity=False, flags=FLAGS):
    """SyntheticTrainStep.step without the optimizer -> Step(losses [B,8], T [B,4,4], pooled [B,512], {name: grad},
    objective).

    flags: the ICP loss bits (DELORA_LOSS_* / DELORA_NORMAL_LINEAR) the step's losses use; lambda_po2pl is cfg's.
    w_pre > 0: the reference's two-resolution recipe through the mirror -- Preprocesser.preprocess_scans in memory (the
    offline stage's row-major point and normal lists), ops.project at W and ops.grids_from_projection
    (Deployer.step); otherwise ops.project + ops.normals at W.  Then OdometryModel's training forward (TensorCoreEncoder
    with autograd, torch heads), GeometryHandler's quaternion -> T and the fused ICP losses.  The objective is their
    mean over the pairs, or with identity that of unsupervised_at_start: False (delora_b200/deploy/deployer.py:206-210),
    MSELoss(T_{B-1}, I) / B."""
    from delora_b200.deploy.deployer import _FusedIcp
    from delora_b200.models.model_parts import GeometryHandler
    ds = cfg["kitti"]
    h, w = ds["vertical_cells"], ds["horizontal_cells"]
    hf, vf = tuple(cfg["horizontal_field_of_view"]), tuple(ds["vertical_field_of_view"])
    b = pts.shape[0] // 2
    if w_pre > 0:
        plist, nlist, lens = _preprocessed_lists(cfg, pts, counts, w_pre)
        image, imap = ops.project(plist, lens, h, w, hf, vf)
        pg, ng = ops.grids_from_projection(plist, nlist, imap)
    else:
        image, _ = ops.project(pts, counts, h, w, hf, vf)
        _, pg, ng = ops.normals(image, ds["neighborhood_side_length"], cfg["epsilon_range"],
                                cfg["min_num_points_in_neighborhood_to_determine_point_class"], grids=True)
    img1, img2 = image[:b].contiguous(), image[b:].contiguous()
    with torch.no_grad():
        pooled = m._tensor_core_path().pooled_features(img1, img2)
    m.zero_grad(set_to_none=True)
    trans, quat = m(image_1=img1, image_2=img2)
    T = GeometryHandler.get_transformation_matrix_quaternion(trans.float(), quat.float(), DEV)
    total, parts = _FusedIcp.apply(T, pg[b:].contiguous(), ng[b:].contiguous(), pg[:b].contiguous(),
                                   ng[:b].contiguous(), (h, w, hf, vf), float(cfg["lambda_po2pl"]), flags,
                                   ops.icp_scratch(b, h * w, pts.device))
    if identity:
        eye = torch.eye(4, device=DEV).view(1, 4, 4)
        loss = torch.nn.MSELoss()(T[-1:], eye) / b
    else:
        loss = total.mean()
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    return Step(parts.detach(), T.detach(), pooled, grads, loss.item())


def grad_dict(flat, cfg):
    from delora_b200.deploy import export
    return export.unpack_blob(flat.cpu().numpy(), cfg)


def _is_tail(name):
    return name.startswith("resnet.fc") or name.startswith("fully_connected")


def grad_spread(c_grads, py_grads):
    """-> (worst relative error of the tail tensors, of the trunk tensors), relative to each tensor's max-abs."""
    worst = {True: 0.0, False: 0.0}
    for k, ref in py_grads.items():
        ref = ref.cpu()
        scale = ref.abs().max().item()
        assert scale > 0, f"{k}: zero gradient in the Python step"
        err = (c_grads[k] - ref).abs().max().item() / scale
        worst[_is_tail(k)] = max(worst[_is_tail(k)], err)
    return worst[True], worst[False]


def rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def build_example(name, out_dir, link):
    """nvcc examples/<name>.c against include/delora_b200.h: link=False compiles it with -Wall -Werror to an object,
    link=True links an executable against the built libdelora_b200.so.  -> the output path."""
    from delora_b200 import build
    nvcc = build._nvcc()
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")
    cmd = [nvcc] + ([] if link else ["-c"]) + [os.path.join(ROOT, "examples", f"{name}.c"), "-I",
                                               os.path.join(ROOT, "include"), "-I", cuda_inc]
    if link:
        libdir = os.path.dirname(build.LIB)
        out = os.path.join(out_dir, name)
        cmd += ["-L", libdir, "-ldelora_b200", "-lcudart", "-Xlinker", "-rpath=" + libdir]
    else:
        out = os.path.join(out_dir, f"{name}.o")
        cmd += ["-Xcompiler", "-Wall,-Werror"]
    r = subprocess.run(cmd + ["-o", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return out


def bits(t):
    """A float32 tensor's bits as int32: bit-for-bit comparisons."""
    return t.contiguous().view(torch.int32)


def same(a, b):
    return torch.equal(bits(a), bits(b))


def align(n):
    """n bytes rounded up to a workspace section's 256-byte alignment."""
    return (n + 255) // 256 * 256


def state(ws):
    """A training workspace's (weights, exp_avg, exp_avg_sq, step), copied to the host."""
    st = ws.get_state()
    torch.cuda.synchronize()
    return tuple(t.cpu().clone() for t in st)


def same_state(a, b):
    return all(same(x, y) if x.dtype == torch.float32 else torch.equal(x, y) for x, y in zip(a, b))


def streams_desc(h=64, w=720, S=2, w_pre=0, n_stride=1000):
    """The descriptor of an S-stream workspace, for the host-only queries."""
    return desc(config(h, w, device="cpu"), n_stride, S, w_pre)


Section = collections.namedtuple("Section", "name offset bytes role geometry flags")


def sections(kind, descs):
    """delora_odometry_workspace_sections of kind (a name of _lib.WS_KINDS) over the descriptors descs (one, or each
    geometry's) -> [Section], or None where the library refuses them."""
    from delora_b200 import _lib
    L = _lib.lib()
    k = _lib.WS_KINDS.index(kind)
    arr = (_lib.OdometryDesc * len(descs))(*descs)
    n = L.delora_odometry_workspace_sections(k, arr, len(descs), None, 0)
    if n < 0:
        return None
    out = (_lib.WsSection * n)()
    assert L.delora_odometry_workspace_sections(k, arr, len(descs), out, n) == n
    return [Section(r.name.decode(), r.offset, r.bytes, _lib.WS_ROLES[r.role], r.geometry, r.flags) for r in out]


def train_params(flags=ops.LOSS_PO2PL | ops.LOSS_PL2PL, lr=1e-5):
    from delora_b200 import _lib
    return _lib.OdometryTrainParams(lr=lr, beta1=0.9, beta2=0.999, eps=1e-8, lambda_po2pl=1.0, loss_flags=flags,
                                    nb_h=7, nb_w=11, epsilon_range=0.5, min_neighbors=10)


# ------------------------------------------------------------------------------------------- streams workspaces
SENTINEL = 1234.5          # what the float outputs hold before a streams call writes them; valid holds 7
GUARD = 4096               # guard bytes on each side of a guarded workspace


def stage_ticks(act, n_stride, frame, count=None):
    """Host staging of every tick of S = act.shape[1] streams: frame(k, s) -> the points [3, n] stream s is given at
    tick k (an inactive stream too: only `active` keeps it out), count(k, s, n) -> its count (default n)
    -> [(points [S, 3, n_stride], counts [S], active [S])]."""
    out = []
    for k in range(act.shape[0]):
        pts = torch.zeros((act.shape[1], 3, n_stride), dtype=torch.float32)
        counts = torch.zeros((act.shape[1],), dtype=torch.int32)
        for s in range(act.shape[1]):
            f = frame(k, s)
            pts[s, :, :f.shape[1]] = f
            counts[s] = f.shape[1] if count is None else count(k, s, f.shape[1])
        out.append((pts, counts, torch.from_numpy(act[k].astype(np.int32))))
    return out


def recipe_pattern(S, ticks=7):
    """The adapting and recipe streams' activity: active [ticks, S] with an inactive stream at tick 1, an idle tick 4
    and stream 0 out at tick 6, the (tick, stream) with an empty frame and the resets {tick: [streams]}."""
    act = np.ones((ticks, S), dtype=bool)
    act[1, S - 1] = False
    act[4, :] = False
    if ticks > 6:
        act[6, 0] = False
    return act, {(2, 1 % S)}, {3: [0]}


def recipe_ticks(pool, S, n_stride, act, empty):
    """stage_ticks of stream s on pool[(3 s + k) % len(pool)] at tick k, an inactive one on another pool frame with its
    real count (only the mask keeps it out), the frames in `empty` with count 0."""
    return stage_ticks(act, n_stride, lambda k, s: pool[(3 * s + k + (0 if act[k, s] else 5)) % len(pool)],
                       lambda k, s, n: 0 if (k, s) in empty else n)


def pool_tick(pool, S, n_stride, k, active, offset=0):
    """Tick k of S streams on the device: stream s serves pool[(3 * (s + offset) + k) % len(pool)] where active[s]."""
    pts = torch.zeros((S, 3, n_stride), dtype=torch.float32)
    counts = torch.zeros((S,), dtype=torch.int32)
    for s in range(S):
        f = pool[(3 * (s + offset) + k) % len(pool)]
        pts[s, :, :f.shape[1]] = f
        counts[s] = f.shape[1]
    return pts.to(DEV), counts.to(DEV), torch.tensor(active, dtype=torch.int32, device=DEV)


def group_tick(g, streams, inputs, updates):
    """Every rank's tick of an AdaptingStreamsGroup on its own stream, all enqueued before one synchronisation -> its
    outputs per rank on the host."""
    torch.cuda.synchronize()
    outs = []
    for r, (pts, counts, active) in enumerate(inputs):
        with torch.cuda.stream(streams[r]):
            outs.append(g.push(r, pts, counts, active, update=updates[r]))
    torch.cuda.synchronize()
    return [tuple(t.cpu() for t in o) for o in outs]


def group_status_ok(g):
    return all(int(s.item()) == 0 for s in g.status)


def history(ticks, act, resets):
    """{(k, s): (previous frame, this frame)} of every pair the streams should serve: (points [3, n], count)."""
    pairs, prev = {}, [None] * act.shape[1]
    for k, (p, c, _) in enumerate(ticks):
        for s in resets.get(k, []):
            prev[s] = None
        for s in range(act.shape[1]):
            if not act[k, s]:
                continue
            if prev[s] is not None:
                pairs[(k, s)] = (prev[s], (p[s], c[s]))
            prev[s] = (p[s], c[s])
    return pairs


def guarded_workspace(nbytes):
    """A device workspace of exactly nbytes between GUARD guard bytes on each side, its own bytes all 0xFF (NaN floats)
    -> (workspace, intact), intact() True while no call has written outside it."""
    buf = torch.full((nbytes + 2 * GUARD,), 0xFF, dtype=torch.uint8, device=DEV)
    pattern = torch.arange(GUARD, device=DEV).to(torch.uint8) ^ 0xA5
    buf[:GUARD] = pattern
    buf[GUARD + nbytes:] = pattern

    def intact():
        torch.cuda.synchronize()
        return torch.equal(buf[:GUARD], pattern) and torch.equal(buf[GUARD + nbytes:], pattern)
    return buf[GUARD:GUARD + nbytes], intact


ROW_WIDTH = {"losses": ops.LOSS_ROW, "info": ops.INFO_ROW, "factor": None}


class Outputs:
    """The outputs of a streams push in its argument order: T [S, 16], valid [S], then the rows named in `rows` (any of
    "losses" [S, LOSS_ROW], "info" [S, INFO_ROW], "factor" [S], in that order), each between a guard row on either
    side.  Every float holds SENTINEL and valid holds 7 until a call writes them."""

    def __init__(self, S, rows=()):
        assert list(rows) == [r for r in ROW_WIDTH if r in rows], rows
        self.T = torch.empty((S, 16), dtype=torch.float32, device=DEV)
        self.valid = torch.empty((S,), dtype=torch.int32, device=DEV)
        self.guarded = [torch.empty((S + 2,) + ((ROW_WIDTH[r],) if ROW_WIDTH[r] else ()), dtype=torch.float32,
                                    device=DEV) for r in rows]
        self.tensors = (self.T, self.valid) + tuple(g[1:S + 1] for g in self.guarded)
        self.fill()

    def fill(self):
        self.valid.fill_(7)
        for t in (self.T, *self.guarded):
            t.fill_(SENTINEL)

    def snapshot(self, k=None):
        """Synchronises, asserts every guard row still holds SENTINEL -> the outputs copied to the host."""
        torch.cuda.synchronize()
        for g in self.guarded:
            assert bool((g[0] == SENTINEL).all()) and bool((g[-1] == SENTINEL).all()), \
                f"tick {k}: a write outside an output row"
        return tuple(t.cpu().clone() for t in self.tensors)


def run_streams(ws, ticks, rows=(), resets=None, updates=None, loads=None, graph=False, hook=None):
    """Every tick (points [S, 3, n], counts [S], active [S]) through one streams workspace -> per tick the outputs of
    Outputs(S, rows) on the host, plus hook(ws) when given.

    Before tick k: the streams in resets[k] are reset through a mask, then loads[k] is loaded (load_weights).  updates:
    the adapting workspaces' update flag of each tick.  graph: every stream inactive, one push per update value (which
    changes no stream's state), the sentinels restored, then one captured push per update value replays each tick."""
    S = ws.desc.max_batch
    pts = torch.zeros((S, 3, ticks[0][0].shape[2]), dtype=torch.float32, device=DEV)
    counts = torch.zeros((S,), dtype=torch.int32, device=DEV)
    active = torch.zeros((S,), dtype=torch.int32, device=DEV)
    mask = torch.zeros((S,), dtype=torch.int32, device=DEV)
    out = Outputs(S, rows)
    args = (pts, counts, active) + out.tensors
    modes = sorted(set(updates)) if updates is not None else [None]

    def push(u):
        if u is None:
            ws.push(*args)
        else:
            ws.push(*args, update=u)
    graphs = {}
    if graph:
        for u in modes:
            push(u)
        torch.cuda.synchronize()
        out.fill()
        for u in modes:
            graphs[u] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphs[u]):
                push(u)
    got = []
    for k, (p, c, a) in enumerate(ticks):
        if resets and k in resets:
            mask.zero_()
            mask[list(resets[k])] = 1
            ws.reset(mask)
        if loads and k in loads:
            ws.load_weights(loads[k])
        pts.copy_(p)
        counts.copy_(c)
        active.copy_(a)
        u = None if updates is None else updates[k]
        if graph:
            graphs[u].replay()
        else:
            push(u)
        got.append(out.snapshot(k) + ((hook(ws),) if hook else ()))
    return got
