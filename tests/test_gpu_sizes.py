"""-m gpu: the reference's other image sizes (SURVEY.md §0 D5): the preprocessing width 64x2250
(config/config_datasets.yaml:31), DARPA 64x512 and VLP-16 16x720 (scripts/time_network.py:62), plus the encoder at the
bench shape 64x2048.  Same bars as tests/test_gpu_parity.py, the oracle is evaluated on the fly (no goldens)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import delora_oracle as orc
from test_gpu_parity import check_projection

pytestmark = pytest.mark.gpu
DEV = "cuda"

SIZES = [  # name, H, W, w_raw, rings, vfov_deg
    ("pre_64x2250", 64, 2250, 2048, 64, (-24.5, 2.0)),
    ("darpa_64x512", 64, 512, 600, 64, (-24.5, 2.0)),
    ("vlp16_16x720", 16, 720, 800, 16, (-15.0, 15.0)),
]
_cache = {}


def case(name):
    if name not in _cache:
        from delora_b200 import synthetic
        _, h, w, w_raw, rings, vf = next(s for s in SIZES if s[0] == name)
        cfg = synthetic.fov_config(h=h, w=w, vfov_deg=vf)
        s1, s2, _, t_pred = synthetic.make_pair(70, w_raw=w_raw, rings=rings, vfov_deg=vf)
        out = orc.pair_forward_backward(s1, s2, t_pred, cfg)
        _cache[name] = (cfg, h, w, s1, s2, t_pred, out)
    return _cache[name]


@pytest.mark.parametrize("name", [s[0] for s in SIZES])
def test_projection_at_reference_sizes(name, cuda_lib):
    cfg, h, w, s1, s2, _, _ = case(name)
    hf, vf = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
    check_projection(s1, h, w, hf, vf, name + "/scan_1")
    check_projection(s2, h, w, hf, vf, name + "/scan_2")


@pytest.mark.parametrize("name", [s[0] for s in SIZES])
def test_normals_at_reference_sizes(name, cuda_lib):
    from delora_b200 import ops
    cfg, h, w, _, _, _, out = case(name)
    image = out["image_1"]
    n_o, enough, _, aux = orc.compute_normal_vectors(image, return_aux=True)
    nrm = ops.normals(image.to(DEV))
    valid = (image[0, 0] != 0) & (image[0, 1] != 0) & (image[0, 2] != 0)
    n_g = nrm[0].permute(1, 2, 0)[valid.to(DEV)].cpu()
    assert torch.equal((n_g != 0).any(dim=1), enough), "has-normal mask must be exact"
    err = (n_g - n_o).norm(dim=1)[enough]
    ev = aux["eigenvalues"]
    gap = (ev[:, 1] - ev[:, 0]) / ev[:, 2].clamp_min(1e-30)
    q = torch.quantile(err, torch.tensor([0.5, 0.99])).tolist()
    print(f"[{name}] normals |dn| median={q[0]:.2e} p99={q[1]:.2e} max={err.max().item():.2e}")
    assert q[1] <= 1e-6
    assert float(err[gap >= 1e-2].max()) <= 5e-5, "well-conditioned normals (eigen-gap >= 1e-2 of the largest eigenvalue)"
    assert float((err * gap.clamp_max(1e-2)).max()) <= 5e-7, "ill-conditioned ones: error x gap stays bounded"


@pytest.mark.parametrize("name", [s[0] for s in SIZES])
def test_pipeline_losses_at_reference_sizes(name, cuda_lib):
    from delora_b200.pipeline import ScanPairPipeline
    cfg, h, w, s1, s2, t_pred, out = case(name)
    hf, vf = cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"]
    pipe = ScanPairPipeline(1, max(s1.shape[1], s2.shape[1]), h, w, hf, vf, device=DEV)
    pipe.load([s1], [s2], t_pred[None])
    losses, grad_t = pipe.step()
    torch.cuda.synchronize()
    row, g = losses[0].cpu(), grad_t[0].cpu().view(3, 4)
    assert int(row[3]) == out["num_pairs"]
    assert row[1].item() == pytest.approx(out["loss_po2pl"], rel=1e-5)
    assert row[2].item() == pytest.approx(out["loss_pl2pl"], rel=1e-5)
    assert (g - out["grad_T"]).abs().max().item() <= 1e-5 * out["grad_T"].abs().max().item()


def test_preprocesser_at_2250(tmp_path, cuda_lib):
    """The offline stage at its real width (horizontal_cells_preprocessing = 2250, 64 rings): the files written by
    the GPU Preprocesser against the oracle's composition (pinned bit-exact to the reference's Preprocesser at
    16x200, tests/golden/preprocess_16x200.npz)."""
    from delora_b200 import synthetic
    from delora_b200.preprocessing.preprocesser import Preprocesser
    velo = tmp_path / "raw" / "00" / "velodyne"
    velo.mkdir(parents=True)
    s1, _, _, _ = synthetic.make_pair(71, w_raw=2048, rings=64)
    raw = np.concatenate((s1.t().numpy(), np.full((s1.shape[1], 1), 0.5, dtype=np.float32)), axis=1).astype(np.float32)
    raw.tofile(velo / "000000.bin")
    cfg = synthetic.preprocessing_config(tmp_path / "raw", tmp_path / "pre", h=64, w_pre=2250, vfov_deg=(-24.5, 2.0), device=DEV)
    Preprocesser(config=cfg).preprocess_data()
    pts = np.load(tmp_path / "pre" / "00" / "scans" / "000000.npy")
    nrm = np.load(tmp_path / "pre" / "00" / "normals" / "000000.npy")
    scan = torch.from_numpy(raw).t().contiguous()
    img = orc.project_to_img(scan[None], 64, 2250, cfg["horizontal_field_of_view"], cfg["kitti"]["vertical_field_of_view"])[0]
    n_o, enough, p_o = orc.compute_normal_vectors(img)
    assert np.array_equal(pts, p_o.numpy()), "point list at 64x2250"
    assert np.array_equal((nrm != 0).any(axis=1), enough.numpy())
    err = np.linalg.norm(nrm - n_o.numpy(), axis=1)[enough.numpy()]
    assert np.quantile(err, 0.99) <= 1e-6


@pytest.mark.parametrize("h,w,b", [(64, 2048, 2), (64, 512, 1), (16, 720, 1)])
def test_encoder_forward_backward_at_bench_and_reference_shapes(h, w, b, cuda_lib):
    """Tensor-core encoder (default path) against the fp32 torch / cuDNN stack at the bench shape 64x2048 (B = 2) and
    the reference's other sizes: features, pose outputs and all 20 convolution weight gradients."""
    from delora_b200 import ops, synthetic
    from delora_b200.models.model import OdometryModel
    from delora_b200.models.tc_encoder import TensorCoreEncoder
    cfg = synthetic.fov_config(h=h, w=w, device=DEV)
    cfg.update({"pre_feature_extraction": False, "resnet_outputs": 1000, "use_dropout": False, "layers": [2, 2, 2, 2],
                "factor_fewer_resnet_channels": 1, "activation_fct": "tanh", "use_single_mlp_at_output": False,
                "use_tensor_core_encoder": False})
    torch.manual_seed(0)
    model = OdometryModel(cfg).to(DEV)
    enc = TensorCoreEncoder(model)
    g = torch.Generator(device=DEV).manual_seed(1)
    img1 = torch.randn(b, 4, h, w, device=DEV, generator=g) * 5.0
    img2 = torch.randn(b, 4, h, w, device=DEV, generator=g) * 5.0
    sel = torch.randn(b, 512, device=DEV, generator=g)
    model.zero_grad()
    ref_feats = model.forward_features(image_1=img1, image_2=img2)
    (ref_feats[3].mean(dim=(2, 3)) * sel).sum().backward()
    ref = [p.grad.clone() for p in enc.trunk_parameters()]
    with torch.no_grad():
        feats = enc.features(img1, img2)
    for (x, fh, fw), r in zip(feats, ref_feats[:4]):
        cos = F.cosine_similarity(ops.nhwc_to_nchw(x, fh, fw).flatten(), r.detach().flatten(), dim=0).item()
        assert cos > 0.999, cos
    model.zero_grad()
    (enc.pooled_features(img1, img2) * sel).sum().backward()
    cosines = [F.cosine_similarity(p.grad.flatten(), r.flatten(), dim=0).item() for p, r in zip(enc.trunk_parameters(), ref)]
    print(f"[{h}x{w}] weight-gradient cosines: stem {cosines[0]:.5f}, min of the other 19 {min(cosines[1:]):.5f}")
    # The 19 trunk layers stay above 0.999.  The stem's kernels are exact on their own (test_stem_kernels_match_torch:
    # weight gradient within 1e-3 of autograd given the same dZ, input carried with 16 mantissa bits, tanh' evaluated
    # from the pre-activation); its lower END-TO-END cosine is set by the bf16 rounding of the gradient
    # that reaches it through 19 layers: for these random inputs the stem gradient is a small coherent part of a sum of
    # incoherent products, so 2^-9 relative noise in dZ shows up 10x amplified.
    assert len(cosines) == 20 and min(cosines[1:]) > 0.999 and cosines[0] >= 0.99, cosines


@pytest.mark.parametrize("b,h,w", [(1, 8, 256), (2, 16, 180), (1, 64, 720), (2, 64, 2048)])
def test_stem_kernels_match_torch(b, h, w, cuda_lib):
    """csrc/conv_stem.cu alone: forward against torch's convolution of the UNROUNDED input (the stem carries
    bf16(x) + bf16(x - bf16(x))) with bf16 weights, weight gradient against autograd for the same dZ."""
    from delora_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(h + w)
    img1 = torch.randn(b, 4, h, w, device=DEV, generator=g) * 5.0
    img2 = torch.randn(b, 4, h, w, device=DEV, generator=g) * 5.0
    wt = torch.randn(64, 8, 3, 3, device=DEV, generator=g) / 72 ** 0.5
    x16 = ops.images_to_nhwc16(img1, img2)
    wst = torch.empty((3, 64, 64), dtype=torch.bfloat16, device=DEV)
    ops.stem_weight_prep(wt, wst)
    y = ops.stem_fprop(x16, wst, h, w, ops.ACT_TANH)
    x = torch.cat([img1, img2], 1)
    wr = wt.to(torch.bfloat16).float().requires_grad_(True)
    pre = F.conv2d(F.pad(x, (1, 1, 0, 0), mode="circular"), wr, stride=(1, 2), padding=(1, 0))
    assert (ops.nhwc_to_nchw(y, h, w // 2) - torch.tanh(pre)).abs().max().item() <= 4e-3       # bf16 output rounding
    yf = y.float()
    assert torch.equal(yf[:, 1:-1, 0], yf[:, 1:-1, w // 2]) and torch.equal(yf[:, 1:-1, w // 2 + 1], yf[:, 1:-1, 1])
    assert float(yf[:, 0].abs().max()) == 0.0 and float(yf[:, -1].abs().max()) == 0.0
    dz = (torch.randn(b, 64, h, w // 2, device=DEV, generator=g) * 0.5).to(torch.bfloat16).float()
    pre.backward(dz)
    dzp = ops.padded_nhwc_zeros(b, h, w // 2, 64, DEV)
    dzp[:, 1:h + 1, 1:w // 2 + 1] = dz.permute(0, 2, 3, 1).to(torch.bfloat16)
    dzp[:, 1:h + 1, 0] = dzp[:, 1:h + 1, w // 2]
    dzp[:, 1:h + 1, w // 2 + 1] = dzp[:, 1:h + 1, 1]
    dw = ops.stem_wgrad(x16, dzp, h, w, 8)
    assert (dw - wr.grad).abs().max().item() <= 1e-3 * wr.grad.abs().max().item()
    assert F.cosine_similarity(dw.flatten(), wr.grad.flatten(), dim=0).item() > 0.999999
