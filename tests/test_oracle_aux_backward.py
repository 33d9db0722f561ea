"""oracle/pnr_aux_backward.py::render_backward (the hand-derived backward for upstream gradients of all six renderer
outputs, no autograd) against autograd through the oracle and against the gradients the reference produced itself for
a loss on rgb, depth and weights (tests/golden/grad_aux_*.npz).  CPU only."""
import os

import pytest
import torch

import aux_grad_util as au
import golden_util as gu

bw = gu.load_by_path("pnr_backward", os.path.join(gu.ROOT, "oracle", "pnr_backward.py"))
ab = gu.load_by_path("pnr_aux_backward", os.path.join(gu.ROOT, "oracle", "pnr_aux_backward.py"))
rel = au.rel


def manual(case, up):
    cfg = case["cfg"]
    return ab.render_backward(case["rays"], case["noise"], gu.oracle_state(case), case["latent"], case["wc"],
                              case["wf"], cfg["NS"], cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"], up,
                              white_bkgd=bool(cfg["white_bkgd"]))


def random_up(case, seed):
    cfg = case["cfg"]
    R, Kc, K = cfg["SB"] * cfg["B"], cfg["n_coarse"], cfg["n_coarse"] + cfg["n_fine"]
    g = torch.Generator().manual_seed(seed)
    up = dict(d_rgb_coarse=torch.randn(R, 3, generator=g), d_depth_coarse=torch.randn(R, generator=g),
              d_weights_coarse=torch.randn(R, Kc, generator=g))
    if cfg["n_fine"] > 0:
        up.update(d_rgb_fine=torch.randn(R, 3, generator=g), d_depth_fine=torch.randn(R, generator=g),
                  d_weights_fine=torch.randn(R, K, generator=g))
    return {k: v * 1e-2 for k, v in up.items()}


@pytest.mark.parametrize("name,source", [("tiny", "golden"), ("sb2_d", "golden"), ("tiny", "random"),
                                         ("sb2_d", "random"), ("ns1_coarse_only", "random")])
def test_render_backward_equals_autograd(name, source):
    case = gu.load_case(name)
    cfg = case["cfg"]
    R = cfg["SB"] * cfg["B"]
    up = au.flat_up(au.load(name), R) if source == "golden" else random_up(case, 11)
    lat = case["latent"].clone().requires_grad_(True)
    wc = {k: v.clone().requires_grad_(True) for k, v in case["wc"].items()}
    wf = None if case["wf"] is None else {k: v.clone().requires_grad_(True) for k, v in case["wf"].items()}
    res = gu.oracle.render(case["rays"], case["noise"], gu.oracle_state(case), lat, wc, wf, cfg["NS"],
                           cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"], white_bkgd=bool(cfg["white_bkgd"]),
                           eval_batch_size=cfg["eval_batch_size"])
    outs, grads = [], []
    for p in ("coarse", "fine") if cfg["n_fine"] > 0 else ("coarse",):
        for q in ("rgb", "depth", "weights"):
            outs.append(res[p][q])
            grads.append(up[f"d_{q}_{p}"])
    torch.autograd.backward(outs, grad_tensors=grads)
    g_c, g_f, d_lat = manual(case, up)
    assert rel(d_lat, lat.grad) < 2e-5
    for k, v in wc.items():
        assert rel(g_c[k], v.grad) < 2e-5, ("coarse", k)
    if wf is not None:
        for k, v in wf.items():
            assert rel(g_f[k], v.grad) < 2e-5, ("fine", k)


@pytest.mark.parametrize("name", au.CASE_NAMES)
def test_render_backward_equals_reference_gradients(name):
    case, aux = gu.load_case(name), au.load(name)
    cfg = case["cfg"]
    g_c, g_f, d_lat = manual(case, au.flat_up(aux, cfg["SB"] * cfg["B"]))
    assert rel(d_lat, aux["g_latent"]) < 1e-4
    for k, v in aux["gc"].items():
        assert rel(g_c[k], v) < 1e-4, ("coarse", k)
    for k, v in aux["gf"].items():
        assert rel(g_f[k], v) < 1e-4, ("fine", k)


@pytest.mark.parametrize("name", au.CASE_NAMES)
def test_aux_terms_reach_the_mlps(name):
    """The fixture is not vacuous: the alpha / depth / weights terms change the reference's gradients well beyond the
    tolerances above, compared with the rgb-only loss of the same inputs and target (tests/golden/grad_*.npz)."""
    aux, rgb_only = au.load(name), gu.load_grad_case(name)
    assert torch.equal(aux["rgb_gt"], rgb_only["rgb_gt"])
    for k in ("lin_out.weight", "blocks.4.fc_0.weight", "blocks.4.fc_1.weight"):
        assert rel(aux["gf"][k], rgb_only["gf"][k]) > 1e-2, ("fine", k)
    assert rel(aux["gc"]["blocks.4.fc_1.weight"], rgb_only["gc"]["blocks.4.fc_1.weight"]) > 1e-2
    assert rel(aux["g_latent"], rgb_only["g_latent"]) > 1e-2


def test_rgb_only_upstream_reproduces_train_loss_backward():
    """render_backward with only the rgb MSE gradients is train_loss_backward."""
    case = gu.load_case("sb2_d")
    cfg = case["cfg"]
    gt = gu.load_grad_case("sb2_d")["rgb_gt"]
    _, o_c, o_f, o_lat = bw.train_loss_backward(case["rays"], gt, case["noise"], gu.oracle_state(case),
                                                case["latent"], case["wc"], case["wf"], cfg["NS"], cfg["n_coarse"],
                                                cfg["n_fine"], cfg["n_fine_depth"], white_bkgd=bool(cfg["white_bkgd"]))
    res = gu.oracle_render(case)
    gtf = gt.reshape(-1, 3)
    up = dict(d_rgb_coarse=2.0 * (res["coarse"]["rgb"] - gtf) / gtf.numel(),
              d_rgb_fine=2.0 * (res["fine"]["rgb"] - gtf) / gtf.numel())
    g_c, g_f, d_lat = manual(case, up)
    assert rel(d_lat, o_lat) < 1e-6
    for k in o_c:
        assert rel(g_c[k], o_c[k]) < 1e-6 and rel(g_f[k], o_f[k]) < 1e-6, k
