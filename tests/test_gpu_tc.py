"""GPU parity of the tensor engine (wgmma split-fp16 fused kernel) against the CPU oracle.
Tolerance on RGB is the north-star 1e-4; sigma (unbounded) is compared relatively."""
import pytest
import torch

import fine_pass_check as fpc
import golden_util as gu

pytestmark = pytest.mark.gpu

TC_CASES = ["c2_small", "c3_small", "c4_small"]


def _check_status():
    import pnr_native as pn
    st = pn.tc_status()
    assert st == 0, f"tensor engine barrier wait timed out (tag {st})"


@pytest.mark.parametrize("name", TC_CASES)
@pytest.mark.parametrize("P", [40, 300])
def test_tc_field_parity(name, P):
    """PixelNeRFNet.forward through the tensor engine: partial tile (40 points) and several
    tiles with a ragged tail (300 points)."""
    import gpu_util
    case = gu.load_case(name)
    cfg = case["cfg"]
    net = gpu_util.build_net(case, engine="tc")
    g = torch.Generator().manual_seed(P)
    xyz = (torch.rand(cfg["SB"], P, 3, generator=g) - 0.5) * 2.4
    dirs = torch.nn.functional.normalize(torch.randn(cfg["SB"], P, 3, generator=g), dim=-1)
    st = gu.oracle_state(case)
    for coarse, w in ((True, case["wc"]), (False, case["wf"] or case["wc"])):
        with torch.no_grad():
            out = net(xyz.cuda(), coarse=coarse, viewdirs=dirs.cuda())
        _check_status()
        ref = gu.oracle.field_eval(xyz, dirs, st, case["latent"], w, cfg["NS"])
        out = out.cpu()
        assert torch.isfinite(out).all()
        assert (out[..., :3] - ref[..., :3]).abs().max() < 1e-4
        rel = (out[..., 3] - ref[..., 3]).abs() / (1.0 + ref[..., 3].abs())
        assert rel.max() < 5e-4, rel.max()  # sigma is unbounded; the RGB tolerance is the contract


@pytest.mark.parametrize("name", TC_CASES)
def test_tc_render_parity(name):
    import gpu_util
    case = gu.load_case(name)
    res = gpu_util.render_case_cuda(case, engine="tc")
    _check_status()
    ref = gu.oracle_render(case)
    c, rc = res["coarse"], ref["coarse"]
    assert (c["rgb"].cpu() - rc["rgb"]).abs().max() < 1e-4
    assert (c["depth"].cpu() - rc["depth"]).abs().max() < 1e-4
    chk = fpc.check_case(case, res, depth_tol=2e-4)
    print(f"{name} tc: {chk}")


def test_tc_matches_simt_large():
    """Many tiles / persistent loop: 20k points, tensor engine vs the fp32 SIMT engine."""
    import gpu_util
    case = gu.load_case("c2_small")
    cfg = case["cfg"]
    g = torch.Generator().manual_seed(1)
    P = 20000
    xyz = ((torch.rand(1, P, 3, generator=g) - 0.5) * 2.4).cuda()
    dirs = torch.nn.functional.normalize(torch.randn(1, P, 3, generator=g), dim=-1).cuda()
    net = gpu_util.build_net(case, engine="tc")
    with torch.no_grad():
        a = net(xyz, coarse=True, viewdirs=dirs)
        _check_status()
        net.engine = "simt"
        b = net(xyz, coarse=True, viewdirs=dirs)
    assert (a[..., :3] - b[..., :3]).abs().max() < 1e-4
    rel = (a[..., 3] - b[..., 3]).abs() / (1.0 + b[..., 3].abs())
    assert rel.max() < 5e-4


@pytest.mark.parametrize("variant", ["no_fine_mlp", "two_objects", "two_objects_no_fine_mlp"])
def test_tc_variants_vs_oracle(variant):
    """Tensor engine against the ORACLE where the reference's callers reconfigure the model: `net.mlp_fine = None`
    (eval/eval.py:140 -> the coarse MLP serves both passes, models.py:242) and a super-batch of objects (SB = 2,
    train/train.py:-B; here c2_small's two source views become two single-view objects with their own rays)."""
    import gpu_util
    case = dict(gu.load_case("c2_small"))
    cfg = dict(case["cfg"])
    if "no_fine_mlp" in variant:
        case["wf"] = None
    if "two_objects" in variant:
        B = case["rays"].shape[1] // 2
        case["rays"] = case["rays"][:, :2 * B].reshape(2, B, 8).contiguous()
        case["src_poses"] = case["src_poses"].reshape(2, 1, 4, 4).contiguous()
        case["noise"] = {k: v[:2 * B].contiguous() for k, v in case["noise"].items()}
        cfg.update(SB=2, NS=1)
    case["cfg"] = cfg
    res = gpu_util.render_case_cuda(case, engine="tc")
    _check_status()
    ref = gu.oracle_render(case)
    assert (res["coarse"]["rgb"].cpu() - ref["coarse"]["rgb"]).abs().max() < 1e-4
    assert (res["coarse"]["weights"].cpu() - ref["coarse"]["weights"]).abs().max() < 1e-4
    chk = fpc.check_case(case, res, depth_tol=2e-4)
    print(f"{variant} tc: {chk}")
