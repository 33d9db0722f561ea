"""The fine-pass checker (tests/fine_pass_check.py) on CPU: it accepts the oracle's own render, including one whose
importance sample sits on a cdf edge and lands in the other bin than a float64 cdf gives, and rejects each kind of
tampered render for the reason the tampering breaks."""
import numpy as np
import pytest
import torch

import fine_pass_check as fpc
import golden_util as gu


def _render(name, noise=None):
    case = dict(gu.load_case(name))
    if noise is not None:
        case["noise"] = noise
    ref = gu.oracle_render(case)
    return case, {p: {k: v.clone() for k, v in d.items()} for p, d in ref.items()}


def _layer2(case, ref, z_fine=None):
    cfg = case["cfg"]
    c = ref["coarse"]
    return fpc.explain_fine_z(case["rays"], c["z"], c["weights"], c["depth"], case["noise"], cfg["n_coarse"],
                              cfg["n_fine"], cfg["n_fine_depth"], 0.01, ref["fine"]["z"] if z_fine is None else z_fine)


def _layer3(case, z, fine):
    return fpc.check_fine_outputs(case["rays"], z, fine, fpc.case_composite(case))


@pytest.mark.parametrize("name", ["tiny", "sb2_d"])
def test_oracle_render_is_accepted(name):
    case, ref = _render(name)
    assert _layer2(case, ref) == 0
    errs = _layer3(case, ref["fine"]["z"], ref["fine"])
    assert max(errs.values()) == 0.0


def test_cdf_edge_flip_is_accepted_and_counted():
    """u put exactly on an fp32 cdf edge that lies below the float64 edge: the fp32 searchsorted takes the upper bin,
    the float64 one the lower, and the checker explains the sample by the admissible upper bin."""
    case, ref = _render("tiny")
    cfg = case["cfg"]
    Kc = cfg["n_coarse"]
    w32 = ref["coarse"]["weights"] + 1e-5
    cdf32 = torch.cumsum(w32 / torch.sum(w32, -1, keepdim=True), -1)          # the oracle's own ops (nerf.py:131-133)
    w64 = ref["coarse"]["weights"].double() + 1e-5
    cdf64 = torch.cumsum(w64 / w64.sum(-1, keepdim=True), -1)
    below = (cdf32[:, :Kc - 1].double() < cdf64[:, :Kc - 1]).nonzero()
    assert below.shape[0] > 0, "no fp32 cdf edge below its float64 value in this case"
    r, i = (int(v) for v in below[0])
    noise = {k: v.clone() for k, v in case["noise"].items()}
    noise["u_fine"][r, 0] = cdf32[r, i]
    case, ref = _render("tiny", noise)
    assert _layer2(case, ref) == 1
    _layer3(case, ref["fine"]["z"], ref["fine"])


def test_sample_moved_to_a_far_bin_is_rejected():
    case, ref = _render("tiny")
    cfg = case["cfg"]
    Kc, Kf, Kfd = cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"]
    r8 = case["rays"].reshape(-1, 8)
    near, far = r8[0, 6], r8[0, 7]
    # importance sample 0 of ray 0 moved by Kc / 2 bins, then re-merged
    u, uj = case["noise"]["u_fine"][:1, :1], case["noise"]["u_fine_jit"][:1, :1]
    z_old = gu.oracle.sample_fine(r8[:1], ref["coarse"]["weights"][:1], u, uj, Kc)[0, 0]
    i = int(torch.round((z_old - near) / (far - near) * Kc - uj[0, 0]))
    s = ((i + Kc // 2) % Kc + uj[0, 0]) / Kc
    z_new = near * (1 - s) + far * s
    assert (z_new - z_old).abs() > 0.4 * (far - near)
    z = ref["fine"]["z"].clone()
    row = z[0].tolist()
    row.remove(float(z_old))
    z[0] = torch.tensor(sorted(row + [float(z_new)]))
    assert Kf - Kfd > 0
    with pytest.raises(AssertionError, match="ray 0: importance sample .* not the sample of any bin"):
        _layer2(case, ref, z)


def test_swapped_samples_are_rejected():
    case, ref = _render("tiny")
    z = ref["fine"]["z"].clone()
    r, k = 5, 7
    z[r, k], z[r, k + 1] = z[r, k + 1].clone(), z[r, k].clone()
    assert z[r, k] != z[r, k + 1]
    with pytest.raises(AssertionError, match="ray 5: merged samples are not sorted"):
        _layer2(case, ref, z)


def test_depth_sample_one_ulp_off_is_rejected():
    case, ref = _render("tiny")
    r8 = case["rays"].reshape(-1, 8)
    zd = gu.oracle.sample_fine_depth(r8, ref["coarse"]["depth"], case["noise"]["n_depth"], 0.01)
    z = ref["fine"]["z"].clone()
    # the first ray whose first depth-centred sample is unclamped and has a larger neighbour in the merge
    for r in range(z.shape[0]):
        k = int((z[r] == zd[r, 0]).nonzero()[-1])
        bumped = float(np.nextafter(np.float32(zd[r, 0]), np.float32(np.inf)))
        if r8[r, 6] < zd[r, 0] < r8[r, 7] and k + 1 < z.shape[1] and z[r, k + 1] > bumped:
            break
    else:
        raise AssertionError("no unclamped depth-centred sample in this case")
    z[r, k] = bumped
    with pytest.raises(AssertionError, match=f"ray {r}: the coarse or depth-centred sample .* is missing"):
        _layer2(case, ref, z)


def test_rgb_at_perturbed_samples_is_rejected():
    """The fine outputs of the most opaque ray computed at samples where its heaviest sample moved halfway to the
    next: the merged samples still pass, the rgb is caught."""
    case, ref = _render("sb2_d")
    cfg = case["cfg"]
    f = ref["fine"]
    r = int(f["weights"].max(-1).values.argmax())
    k = int(f["weights"][r].argmax())
    zp = f["z"].clone()
    zp[r, k] = 0.5 * (zp[r, k] + zp[r, k + 1])
    w, rgb, dep = fpc.case_composite(case)(case["rays"].reshape(-1, 8), zp, cfg["SB"])
    tampered = dict(f, rgb=rgb, depth=dep, weights=w)
    assert _layer2(case, ref) == 0
    with pytest.raises(AssertionError, match=r"fine rgb of 1 rays \(first: row %d\)" % r):
        _layer3(case, f["z"], tampered)


def test_eps_follows_the_derivation():
    assert fpc.cdf_eps(64) == 132 * 2.0 ** -24
    assert fpc.cdf_eps(512) < 1e-4
