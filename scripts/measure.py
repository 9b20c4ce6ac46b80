"""What the odometry and training measurement scripts share: the card query, the model and its weights, the frames,
graph capture, the three timers, the samples and the JSON output.

A script run as `python scripts/<name>.py` has this directory on sys.path and imports this module as `measure`; the
scripts import nothing from each other.
"""
import ctypes
import json
import math
import os
import statistics
import subprocess
import time

import torch

from delora_b200 import synthetic
from delora_b200.deploy import export
from delora_b200.models.model import OdometryModel

DEV = "cuda:0"
GPU_QUERY = "name, power.limit, clocks.sm, clocks.max.sm"

# the two sensor geometries (H, W, w_pre) of the adapting streams of several geometries, and the streams per geometry
GEOMS = ((64, 720, 2250), (64, 512, 512))
GEOMS_STREAMS = (1, 4)


def gpu_info():
    """The current device's nvidia-smi line of GPU_QUERY, or "unavailable" when the query fails."""
    cmd = ["nvidia-smi", "--query-gpu=" + GPU_QUERY.replace(" ", ""), "--format=csv,noheader"]
    try:
        r = subprocess.run(cmd, capture_output=True, text=True)
    except OSError:
        return "unavailable"
    lines = r.stdout.strip().splitlines() if r.returncode == 0 else []
    i = torch.cuda.current_device()
    return lines[i] if i < len(lines) else "unavailable"


def model_config(h, w, vfov=synthetic.KITTI_VFOV_DEG):
    """synthetic.fov_config at h x w on DEV, with the model every script measures: tanh, two heads, layers [2, 2, 2, 2],
    1000 ResNet outputs, no dropout."""
    cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vfov, device=DEV)
    cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                "use_dropout": False})
    return cfg


def _seeded_model(cfg):
    torch.manual_seed(0)
    return OdometryModel(cfg).to(DEV).eval()


def _blob(model, cfg):
    return torch.from_numpy(export.pack_state_dict(model.state_dict(), cfg)).to(DEV)


def untrained_blob(cfg):
    """The packed weights, on DEV, of OdometryModel(cfg) as torch.manual_seed(0) initialises it."""
    return _blob(_seeded_model(cfg), cfg)


def near_identity_blob(cfg):
    """untrained_blob with the heads' last layers scaled by 0.01 and the identity transform as their bias: T near I, as
    after the reference's identity pre-training.  The dense ICP's work depends on T, and untrained heads give a T far
    from the truth."""
    model = _seeded_model(cfg)
    with torch.no_grad():
        for head, bias in ((model.fully_connected_rotation, [0.0, 0.0, 0.0, 1.0]),
                           (model.fully_connected_translation, [0.0, 0.0, 0.0])):
            head[3].weight.mul_(0.01)
            head[3].bias.copy_(torch.tensor(bias))
    return _blob(model, cfg)


def pairs(h, count):
    """Synthetic scan pairs 0 .. count - 1 with h rings of 2048 columns: [(scan_1, scan_2), ...]."""
    return [synthetic.make_pair(i, w_raw=2048, rings=h)[:2] for i in range(count)]


def n_stride(pairs):
    """The most points of any scan of `pairs`."""
    return max(max(a.shape[1], b.shape[1]) for a, b in pairs)


def staged(scans, n_stride):
    """-> (points [len(scans), 3, n_stride] float32, zero-padded; counts [len(scans)] int32), both on DEV."""
    pts = torch.zeros((len(scans), 3, n_stride), dtype=torch.float32)
    for i, s in enumerate(scans):
        pts[i, :, :s.shape[1]] = s
    counts = torch.tensor([s.shape[1] for s in scans], dtype=torch.int32)
    return pts.to(DEV), counts.to(DEV)


def geom_desc(cfg, h, w, w_pre, n_stride, S):
    """The descriptor of cfg's model at h x w with normals at w_pre, for S streams or pairs of up to n_stride points."""
    c = dict(cfg, kitti=dict(cfg["kitti"], vertical_cells=h, horizontal_cells=w))
    d = export.desc_from_config(c, "kitti", n_stride, S)
    d.w_pre = w_pre
    return d


def capture(fn, warmup, stream=None):
    """fn run `warmup` times (first frames, the launchers' host-side state), a device synchronise, then fn captured
    into a CUDA graph, on `stream` when one is given."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=stream):
        fn()
    return g


def events_ms(fn, *, seconds=None, calls=None):
    """-> (ms per call of fn, calls timed), from CUDA events on the current stream around back-to-back calls.

    calls=n: around n calls.  seconds=s: 10 warm-up calls, a 10-call estimate, then around at least 50 calls and at
    least s seconds of work."""
    assert (seconds is None) != (calls is None), "events_ms takes seconds or calls"
    if seconds is not None:
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        est, _ = events_ms(fn, calls=10)
        calls = max(50, math.ceil(seconds * 1e3 / max(est, 1e-3)))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / calls, calls


def host_ms(fn, seconds, devices, every, warmup):
    """ms per call of fn from the host clock: `warmup` calls and a synchronise of `devices`, then calls until at least
    `seconds` have passed, synchronising `devices` every `every` calls.  CUDA events time one device's stream; this
    times work that spans devices."""
    def sync():
        for d in devices:
            torch.cuda.synchronize(d)

    for _ in range(warmup):
        fn()
    sync()
    n, t0 = 0, time.perf_counter()
    while True:
        fn()
        n += 1
        if n % every == 0:
            sync()
            el = time.perf_counter() - t0
            if el >= seconds:
                return el * 1e3 / n


def alternate(sides, samples, timer):
    """{side: [ms, ...]}: `samples` rounds, each timing every fn of {side: fn} once with timer(fn), in the dict's order,
    so that drift of the card's clock hits every side alike."""
    out = {k: [] for k in sides}
    for _ in range(samples):
        for k, fn in sides.items():
            out[k].append(timer(fn))
    return out


def summary(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def paired(xs, ys):
    """-> (the differences y - x of paired samples, their median)."""
    d = [y - x for x, y in zip(xs, ys)]
    return d, statistics.median(d)


def emit(res, path=None):
    """Print res as JSON (indent 1) and, when `path` is given, write the same text there."""
    text = json.dumps(res, indent=1)
    print(text)
    if path:
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        with open(path, "w") as f:
            f.write(text)


def enable_peer_access(n):
    """Peer access both ways between devices 0 .. n-1, in the CUDA runtime that libdelora_b200.so loaded."""
    from delora_b200 import _lib
    _lib.lib()
    cudart = ctypes.CDLL("libcudart.so.12")
    for i in range(n):
        torch.cuda.set_device(i)
        for j in range(n):
            if i != j:
                rc = cudart.cudaDeviceEnablePeerAccess(j, 0)
                assert rc in (0, 704), f"cudaDeviceEnablePeerAccess({i} -> {j}) failed: {rc}"   # 704: already on
    torch.cuda.set_device(0)
