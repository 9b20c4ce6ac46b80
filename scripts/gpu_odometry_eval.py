"""What evaluation through the C ABI costs on the GPU.

(a) delora_odometry_streams_push_residual against delora_odometry_streams_push, ms per tick at S in {1, 4, 16} for
    64 x 2048 and 64 x 720, all streams active.  Each stream alternates between the two scans of a synthetic pair
    (0.5 m, 1 degree apart), so every tick sees a consecutive frame with a realistic small motion; one captured graph
    holds the two ticks.  The ICP's cost depends on T, and untrained heads give a T far from the truth, so the heads'
    last layers are scaled by 0.01 with the identity quaternion as bias (T near I, as after the reference's identity
    pre-training).
(b) delora_odometry_train_eval against delora_odometry_train_step at B in {1, 4, 16}, same sizes, the same near-identity
    model, w_pre 0, lr 0 (the weights, and so T and the ICP's work, stay put over the replays).

Graph replays timed with CUDA events over at least --seconds of work per sample; the two sides alternate (a, b, a, b,
...) and the medians are reported with every sample.  The card's name, power limit and SM clocks are read in the same
run.  Writes odometry_eval.json to --out.

    python scripts/gpu_odometry_eval.py [--seconds 0.5] [--samples 3] [--out DIR]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from delora_b200 import synthetic  # noqa: E402
from delora_b200.deploy import capi, export  # noqa: E402
from delora_b200.models.model import OdometryModel  # noqa: E402
from gpu_odometry_streams import DEV, gpu_info, staged, time_replays  # noqa: E402

SIZES = ((64, 2048), (64, 720))
BATCHES = (1, 4, 16)


def near_identity_blob(cfg):
    torch.manual_seed(0)
    model = OdometryModel(cfg).to(DEV).eval()
    with torch.no_grad():
        for head, bias in ((model.fully_connected_rotation, [0.0, 0.0, 0.0, 1.0]),
                           (model.fully_connected_translation, [0.0, 0.0, 0.0])):
            head[3].weight.mul_(0.01)
            head[3].bias.copy_(torch.tensor(bias))
    return torch.from_numpy(export.pack_state_dict(model.state_dict(), cfg)).to(DEV)


class Ticks:
    """One streams workspace (plain or residual) and a graph of two ticks: every stream's scan_1, then its scan_2."""

    def __init__(self, cfg, blob, pairs, n_stride, residual):
        S = len(pairs)
        d = export.desc_from_config(cfg, "kitti", n_stride, S)
        self.ws = (capi.ResidualStreamsWorkspace(d, blob, capi.residual_params(cfg)) if residual
                   else capi.StreamsWorkspace(d, blob))
        self.frames = [staged([p[i] for p in pairs], n_stride) for i in (0, 1)]
        self.active = torch.ones((S,), dtype=torch.int32, device=DEV)
        self.T = torch.zeros((S, 16), dtype=torch.float32, device=DEV)
        self.valid = torch.zeros((S,), dtype=torch.int32, device=DEV)
        self.out = (self.T, self.valid) + ((torch.zeros((S, 8), dtype=torch.float32, device=DEV),) if residual else ())
        self.two_ticks()                 # first frames cached; warms the launchers' host-side state
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.two_ticks()

    def two_ticks(self):
        for pts, counts in self.frames:
            self.ws.push(pts, counts, self.active, *self.out)


class Train:
    """One training workspace and a graph of one step or one eval on B pairs."""

    def __init__(self, cfg, blob, pairs, n_stride, evaluate):
        B = len(pairs)
        d = export.desc_from_config(cfg, "kitti", n_stride, B)
        d.w_pre = 0
        self.ws = capi.TrainingWorkspace(d, blob, capi.train_params(cfg, 0.0))
        self.pts, self.counts = staged([p[0] for p in pairs] + [p[1] for p in pairs], n_stride)
        self.call = self.ws.eval if evaluate else self.ws.step
        self.call(self.pts, self.counts)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.result = self.call(self.pts, self.counts)


def alternate(a, b, seconds, samples):
    """-> (samples of a, samples of b) in ms per replay, taken a, b, a, b, ..."""
    xs, ys = [], []
    for _ in range(samples):
        xs.append(time_replays(a.graph.replay, seconds)[0])
        ys.append(time_replays(b.graph.replay, seconds)[0])
    return xs, ys


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5)
    ap.add_argument("--samples", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    res = {"gpu_before": gpu_info(), "gpu_query": "name, power.limit, clocks.sm, clocks.max.sm",
           "seconds_per_sample": args.seconds, "sizes": {}}
    for h, w in SIZES:
        cfg = synthetic.fov_config(h=h, w=w, device=DEV)
        cfg.update({"activation_fct": "tanh", "use_single_mlp_at_output": False, "layers": [2, 2, 2, 2],
                    "resnet_outputs": 1000, "pre_feature_extraction": False, "factor_fewer_resnet_channels": 1,
                    "use_dropout": False})
        blob = near_identity_blob(cfg)
        pairs_all = [synthetic.make_pair(i, w_raw=2048, rings=h)[:2] for i in range(max(BATCHES))]
        n_stride = max(max(a.shape[1], b.shape[1]) for a, b in pairs_all)
        streams, train = {}, {}
        for n in BATCHES:
            pairs = pairs_all[:n]
            plain, scored = Ticks(cfg, blob, pairs, n_stride, False), Ticks(cfg, blob, pairs, n_stride, True)
            xs, ys = alternate(plain, scored, args.seconds, args.samples)
            torch.cuda.synchronize()
            ms_p, ms_r = statistics.median(xs) / 2, statistics.median(ys) / 2       # two ticks per replay
            streams[n] = {"push_ms_per_tick": ms_p, "push_residual_ms_per_tick": ms_r, "added_ms_per_tick": ms_r - ms_p,
                          "push_samples_ms": [x / 2 for x in xs], "push_residual_samples_ms": [y / 2 for y in ys],
                          "T_bit_identical": bool(torch.equal(plain.T, scored.T)) and bool(scored.valid.all()),
                          "losses_last_tick": scored.out[2].cpu().tolist(),
                          "workspace_MiB": [plain.ws.workspace.numel() / 2**20, scored.ws.workspace.numel() / 2**20]}
            del plain, scored
            torch.cuda.empty_cache()
            step, ev = Train(cfg, blob, pairs, n_stride, False), Train(cfg, blob, pairs, n_stride, True)
            xs, ys = alternate(step, ev, args.seconds, args.samples)
            torch.cuda.synchronize()
            train[n] = {"train_step_ms": statistics.median(xs), "train_eval_ms": statistics.median(ys),
                        "train_step_samples_ms": xs, "train_eval_samples_ms": ys,
                        "outputs_bit_identical": all(bool(torch.equal(a, b)) for a, b in zip(step.result[:3], ev.result))}
            del step, ev
            torch.cuda.empty_cache()
        res["sizes"][f"{h}x{w}"] = {"n_stride": n_stride, "streams_S": streams, "train_B": train}
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "odometry_eval.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
