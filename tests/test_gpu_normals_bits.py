"""-m gpu: the 7x11 normals kernels give the same bits as they always have.

tests/golden/normals_bits.json holds SHA-256 digests of every output of delora_project_normals_fwd (image, index_map,
pts_grid, nrm_grid) and of delora_normals_fwd (normals, pts_grid, nrm_grid), taken from a build before the tap loop
became predicated and the Jacobi sweep branch-free.  The cases cover the bench batch (8 pairs of 64x2048, C = 3, the
pairs bench.py times first), four channels, edge tiles on both borders, an empty scan and a one-tile-high image.

Run as a script to write the digests of whichever build it imports:
    python tests/test_gpu_normals_bits.py --root CHECKOUT --write OUT.json
"""
import hashlib
import json
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "normals_bits.json")


def _batch(clouds, channels):
    """[B, C, N] (NaN past each scan's end, random reflectance as a fourth channel) + counts [B], on the GPU."""
    nmax = max([c.shape[1] for c in clouds] + [1]) + 3
    pts = torch.full((len(clouds), channels, nmax), float("nan"))
    gen = torch.Generator().manual_seed(0)
    for i, c in enumerate(clouds):
        pts[i, :3, :c.shape[1]] = c
        if channels > 3:
            pts[i, 3:, :c.shape[1]] = torch.rand((channels - 3, c.shape[1]), generator=gen)
    return pts.cuda(), torch.tensor([c.shape[1] for c in clouds], dtype=torch.int32).cuda()


def _pairs(k, **kw):
    """Scans of pairs 0..k-1 in the pipeline's order: every scan_1, then every scan_2."""
    from delora_b200 import synthetic
    pairs = [synthetic.make_pair(i, **kw) for i in range(k)]
    return [p[0] for p in pairs] + [p[1] for p in pairs]


def cases():
    """name -> (clouds, channels, h, w, vfov_deg or None for KITTI's)."""
    small = dict(w_raw=192, rings=16, vfov_deg=(-15.0, 15.0))
    s = _pairs(2, **small)
    return {
        "bench_8x64x2048_c3": (_pairs(8, w_raw=2048), 3, 64, 2048, None),
        "16x180_c4": (s, 4, 16, 180, (-15.0, 15.0)),
        "16x180_c3_empty_scan": ([s[0], torch.zeros((3, 0)), s[1]], 3, 16, 180, (-15.0, 15.0)),
        "8x64_c3": (s, 3, 8, 64, (-15.0, 15.0)),
        "20x100_c3": (_pairs(1, w_raw=128, rings=24, vfov_deg=(-15.0, 15.0)), 3, 20, 100, (-15.0, 15.0)),
    }


def _sha(t):
    return hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def digests():
    """{case: {output: sha256}}; also checks that the depth keys are all-ones after two calls in a row."""
    from delora_b200 import ops, synthetic
    out = {}
    for name, (clouds, channels, h, w, vfov) in cases().items():
        cfg = synthetic.fov_config(h=h, w=w, **({} if vfov is None else {"vfov_deg": vfov}))
        hf, vf = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
        pts, n = _batch(clouds, channels)
        first = ops.project_normals(pts, n, h, w, hf, vf)
        image, imap, pg, ng = ops.project_normals(pts, n, h, w, hf, vf)
        torch.cuda.synchronize()
        for a, b in zip(first, (image, imap, pg, ng)):
            assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), name
        assert bool((ops._keys(pts.device, pts.shape[0], h * w) == -1).all()), f"{name}: keys not all-ones"
        out[name] = {"image": _sha(image), "index_map": _sha(imap), "pts_grid": _sha(pg), "nrm_grid": _sha(ng)}
        # the same image through delora_normals_fwd (normals_7x11_kernel)
        nrm, pg2, ng2 = ops.normals(image, (7, 11), 0.5, 10, grids=True)
        torch.cuda.synchronize()
        out[name + "/normals_fwd"] = {"normals": _sha(nrm), "pts_grid": _sha(pg2), "nrm_grid": _sha(ng2)}
    return out


def test_normals_bits_match_golden(cuda_lib):
    with open(GOLDEN) as f:
        want = json.load(f)
    got = digests()
    assert sorted(got) == sorted(want)
    for name in want:
        assert got[name] == want[name], name


if __name__ == "__main__":
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(HERE))
    ap.add_argument("--write", required=True)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    d = digests()
    with open(args.write, "w") as f:
        json.dump(d, f, indent=1, sort_keys=True)
    import delora_b200
    print("digests of", os.path.dirname(delora_b200.__file__), "->", args.write)
