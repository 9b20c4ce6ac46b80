"""The float64 normals reference and its checker (tests/normals_reference.py), on the CPU: its gate and counts equal the
oracle's, the 7x11 kernels' fp32 covariance formation (restated in numpy) stays inside terms 1-3 of the bound, and the
checker accepts the float64 answer rounded to fp32 but rejects wrong eigenvectors, rotations beyond the bound, flipped
orientations, wrong mask bits and NaN normals."""
import numpy as np
import pytest
import torch

import normals_reference as NR
from oracle import delora_oracle as orc

FAMILIES = NR.families()
FAMILY_IDS = [f.name for f in FAMILIES]


def _oracle_aux(img, nb, eps, min_nb):
    _, enough, _, aux = orc.compute_normal_vectors(torch.from_numpy(np.ascontiguousarray(img))[None], nb, eps, min_nb,
                                                   return_aux=True)
    return enough.numpy(), aux["number_neighbours"].numpy(), aux["pixel_index"].numpy()


def _mask_and_counts_match(img, nb, eps, min_nb):
    ref = NR.reference(img, nb, eps, min_nb)
    enough, count, pix = _oracle_aux(img, nb, eps, min_nb)
    assert np.array_equal(np.nonzero(ref.valid)[0], pix)
    assert np.array_equal(ref.count[pix], count)
    assert np.array_equal(ref.has[pix], enough)


@pytest.mark.parametrize("fam", FAMILIES, ids=FAMILY_IDS)
def test_mask_and_counts_equal_the_oracle(fam):
    for img in fam.images:
        _mask_and_counts_match(img, (7, 11), fam.eps, fam.min_nb)


@pytest.mark.parametrize("name", ["small_16x180", "kitti_64x720"])
def test_mask_and_counts_on_the_goldens(name, golden):
    from helpers import case_inputs
    meta = golden[name]
    cfg, (scan_1, _, _, _) = case_inputs(meta)
    image = orc.project_to_img(scan_1[None], meta["H"], meta["W"], cfg["horizontal_field_of_view"],
                               cfg["kitti"]["vertical_field_of_view"])[0]
    img = image[0, :3].numpy()
    _mask_and_counts_match(img, (7, 11), 0.5, 10)
    _mask_and_counts_match(img, (5, 9), 0.5, 10)


def test_gate_family_hits_its_edges():
    """The F5 images put centres at exactly min_nb - 1 and min_nb neighbours and count the |dr| = eps taps."""
    for fam in NR.family_gate():
        ref = NR.reference(fam.images[0], (7, 11), fam.eps, fam.min_nb)
        w = fam.images[0].shape[2]
        counts = {(ci, cj): int(ref.count[(7 * ci + 3) * w + 11 * cj + 5]) for ci in range(2) for cj in range(3)}
        assert counts[(0, 0)] == fam.min_nb - 1 and counts[(0, 1)] == fam.min_nb, (fam.name, counts)
        assert counts[(0, 2)] == 1 + 12, (fam.name, counts)
        assert counts[(1, 0)] == 1 + 6 + (4 if fam.eps > 0 else 0), (fam.name, counts)


@pytest.mark.parametrize("fam", FAMILIES, ids=FAMILY_IDS)
def test_fp32_one_pass_covariance_within_terms_1_to_3(fam):
    worst = 0.0
    for img in fam.images:
        ref = NR.reference(img, (7, 11), fam.eps, fam.min_nb)
        cov, n = NR.restate_7x11_cov(img, fam.eps)
        assert np.array_equal(n, ref.count)
        err = np.sqrt(((cov[ref.pix].astype(np.float64) - ref.C) ** 2).sum(axis=(1, 2)))
        ratio = err / np.maximum(ref.eps_cov, 1e-300)
        assert (ratio <= 1).all(), (fam.name, ratio.max())
        worst = max(worst, float(ratio.max()) if len(ratio) else 0.0)
    print(f"[{fam.name}] fp32 one-pass covariance error / terms 1-3: max {worst:.3f}")


def _planes_ref():
    fam = NR.family_planes()[1]
    img = fam.images[1]
    return img, NR.reference(img, (7, 11), fam.eps, fam.min_nb)


def test_checker_accepts_the_float64_answer_in_fp32():
    for fam in FAMILIES:
        for k, img in enumerate(fam.images):
            ref = NR.reference(img, (7, 11), fam.eps, fam.min_nb)
            vec = NR.oriented_eigvec(ref)
            zero = (ref.C == 0).all(axis=(1, 2))
            vec[zero] = 0
            vec[zero, 0] = -np.sign(ref.pts[ref.pix][zero, 0])
            nv, pg, ng = NR.outputs(ref, vec)
            NR.check(ref, nv, pg, ng, label=f"{fam.name}[{k}]")


def _rejects(ref, nv, pg, ng):
    with pytest.raises(AssertionError):
        NR.check(ref, nv, pg, ng)


def test_checker_rejects_v1():
    _, ref = _planes_ref()
    _rejects(ref, *NR.outputs(ref, NR.oriented_eigvec(ref, 1)))


def test_checker_rejects_a_rotation_by_ten_times_the_bound():
    _, ref = _planes_ref()
    gap = ref.lam[:, 1] - ref.lam[:, 0]
    gapped = gap > 4 * ref.eps
    assert gapped.sum() > 100
    dk = ref.eps / np.where(gapped, gap - ref.eps, 1.0) + NR.EPS_VEC
    ang = np.minimum(10 * dk, np.pi / 2) * gapped
    v0, v1 = ref.V[:, :, 0], ref.V[:, :, 1]
    vec = np.cos(ang)[:, None] * v0 + np.sin(ang)[:, None] * v1
    c = ref.pts[ref.pix]
    vec[(vec * c).sum(axis=1) > 0] *= -1
    one = np.zeros(len(ref.pix), bool)
    one[np.nonzero(gapped)[0][len(np.nonzero(gapped)[0]) // 2]] = True
    good = NR.oriented_eigvec(ref)
    good[one] = vec[one].astype(np.float32)
    _rejects(ref, *NR.outputs(ref, good))


def test_checker_rejects_a_flipped_orientation():
    _, ref = _planes_ref()
    vec = NR.oriented_eigvec(ref)
    vec[len(vec) // 2] *= -1
    _rejects(ref, *NR.outputs(ref, vec))


def test_checker_rejects_a_flipped_mask_bit():
    _, ref = _planes_ref()
    nv, pg, ng = NR.outputs(ref, NR.oriented_eigvec(ref))
    ng[ref.pix[3], 3] = 0.0
    _rejects(ref, None, pg, ng)
    nv, pg, ng = NR.outputs(ref, NR.oriented_eigvec(ref))
    off = np.nonzero(~ref.has)[0][0]
    ng[off, 3] = 1.0
    _rejects(ref, None, pg, ng)


def test_checker_rejects_a_nan_normal():
    _, ref = _planes_ref()
    vec = NR.oriented_eigvec(ref)
    vec[7] = np.nan
    _rejects(ref, *NR.outputs(ref, vec))


def test_checker_rejects_a_point_grid_bit():
    _, ref = _planes_ref()
    nv, pg, ng = NR.outputs(ref, NR.oriented_eigvec(ref))
    pg[ref.pix[0], 3] = np.array(ref.pix[0] + 1, np.int32).view(np.float32)
    _rejects(ref, nv, pg, ng)


def test_isolated_pixels_have_no_normal_at_any_min_neighbors():
    fam = NR.family_degenerate()[0]
    iso = fam.images[2]
    for mn in (0, 1, 2):
        ref = NR.reference(iso, (7, 11), 0.5, mn)
        alone = ref.valid & (ref.count == 1)
        assert alone.sum() == 7 and not ref.has[alone].any()
        corner = ref.shape[0] * ref.shape[1] - 1          # the clamp repeats it: 4 x 6 taps of the same point
        assert ref.count[corner] == 24 and ref.has[corner] and (ref.C == 0).all()
