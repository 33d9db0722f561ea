"""The CUDA sources of the SIMT path executed on the CPU by the host emulator of tests/cuda_emu: first the
GPU-validated forward kernels against the oracle (this checks the emulator), then `pnr_field_backward` -- which has
not run on a GPU yet -- against the hand-derived oracle backward and the reference's own gradients."""
import os

import pytest
import torch

import emu_util as eu
import fine_pass_check as fpc
import golden_util as gu

bw = gu.load_by_path("pnr_backward", os.path.join(gu.ROOT, "oracle", "pnr_backward.py"))


def rel(a, ref):
    return ((a - ref).abs().max() / (ref.abs().max() + 1e-20)).item()


@pytest.mark.parametrize("name", ["tiny", "sb2_d"])
def test_emulated_forward_field_matches_reference_fixture(name):
    case = gu.load_case(name)
    cfg, ref = case["cfg"], case["ref"]
    keep = []
    scene = eu.scene_struct(case, gu.oracle_state(case), keep)
    mlp = eu.mlp_struct(case["wc"], cfg["d_hidden"])
    xyz, dirs = ref["field_xyz"].contiguous(), ref["field_dirs"].contiguous()
    SB, P = xyz.shape[0], xyz.shape[1]
    out = torch.empty(SB, P, 4)
    L = eu.lib()
    nbytes = L.pnr_field_workspace_bytes(scene, mlp, P, 1)
    ws = torch.empty(nbytes, dtype=torch.uint8)
    eu.ok(L.pnr_field_eval(scene, mlp, eu.ptr(xyz), eu.ptr(dirs), eu.ptr(out), P, 1, ws.data_ptr(), nbytes, None))
    err = (out - ref["field_coarse"]).abs() / (1.0 + ref["field_coarse"].abs())
    assert err.max() < 5e-5


@pytest.mark.parametrize("name", ["tiny", "tiny_sb2", "sb2_d", "ns1_coarse_only"])
def test_emulated_render_matches_oracle(name):
    """pnr_render (sample -> field -> composite -> resample -> sort -> field -> composite) on the emulator, same
    assertions as tests/test_gpu_parity.py::test_render_parity.  sb2_d (two objects, visible in both passes) is so far
    only covered here."""
    case = gu.load_case(name)
    loss, _, _, _, t = _emulated_training_step(case, torch.zeros(case["cfg"]["SB"], case["cfg"]["B"], 3),
                                                backward=False)
    ref = gu.oracle_render(case)
    assert (t["z_coarse"] - ref["coarse"]["z"]).abs().max() < 1e-6
    assert (t["rgb_coarse"] - ref["coarse"]["rgb"]).abs().max() < 1e-4
    assert (t["depth_coarse"] - ref["coarse"]["depth"]).abs().max() < 1e-4
    assert (t["weights_coarse"] - ref["coarse"]["weights"]).abs().max() < 1e-4
    if case["cfg"]["n_fine"] > 0:
        fine_checked(case, t)


@pytest.mark.parametrize("name,chunk_rows", [("tiny", 0), ("sb2_d", 0), ("sb2_d", 24), ("ns1_coarse_only", 0),
                                             ("c2_small", 0), ("c4_small", 48)])
def test_emulated_field_backward_matches_oracle_formulas(name, chunk_rows, monkeypatch):
    """chunk_rows > 0 forces several point chunks (gradient accumulation across chunks); ns1_coarse_only is the
    single-view case (no view mean) with d_hidden = 128; c2_small / c4_small are the shipped d_hidden = 512 with 2 / 3
    views (several SGEMM tiles in every dimension), c4_small with an explicit principal point."""
    if chunk_rows:
        monkeypatch.setenv("PNR_BWD_CHUNK_ROWS", str(chunk_rows))
    case = gu.load_case(name)
    cfg, ref = case["cfg"], case["ref"]
    keep = []
    state = gu.oracle_state(case)
    scene = eu.scene_struct(case, state, keep)
    mlp = eu.mlp_struct(case["wc"], cfg["d_hidden"])
    xyz, dirs = ref["field_xyz"].contiguous(), ref["field_dirs"].contiguous()
    SB, P = xyz.shape[0], xyz.shape[1]
    d_out = torch.randn(SB, P, 4, generator=torch.Generator().manual_seed(5)).contiguous()
    _, sv = bw.field_forward_saved(xyz, dirs, state, case["latent"], case["wc"], cfg["NS"])
    g_ref, dlat_ref, dxyz_ref = bw.field_backward(sv, d_out)
    grads = {k: torch.zeros_like(v) for k, v in case["wc"].items()}
    gs = eu.mlp_struct(grads, cfg["d_hidden"])
    V, Cc, Hl, Wl = case["latent"].shape
    d_lat = torch.zeros(V, Hl, Wl, Cc)
    d_xyz = torch.empty(SB, P, 3)
    L = eu.lib()
    nbytes = L.pnr_field_backward_workspace_bytes(scene, mlp, P)
    ws = torch.empty(nbytes, dtype=torch.uint8)
    eu.ok(L.pnr_field_backward(scene, mlp, eu.ptr(xyz), eu.ptr(dirs), eu.ptr(d_out), gs, eu.ptr(d_lat),
                               eu.ptr(d_xyz), P, ws.data_ptr(), nbytes, None))
    assert dxyz_ref.abs().max() > 0 and dlat_ref.abs().max() > 0 and g_ref["lin_in.weight"].abs().max() > 0
    assert rel(d_xyz, dxyz_ref) < 1e-4
    assert rel(d_lat.permute(0, 3, 1, 2), dlat_ref) < 1e-4
    for k, v in g_ref.items():
        assert rel(grads[k], v) < 1e-4, k


def fine_checked(case, t):
    """Every ray's fine pass against a reference conditioned on the emulated coarse pass (tests/fine_pass_check.py
    layers 2 and 3); returns the number of importance samples that took an admissible non-float64 bin."""
    cfg = case["cfg"]
    coarse = dict(z=t["z_coarse"], weights=t["weights_coarse"], depth=t["depth_coarse"])
    fine = dict(z=t["z_fine"], rgb=t["rgb_fine"], depth=t["depth_fine"], weights=t["weights_fine"])
    res = fpc.check_render(case["rays"], coarse, fine, case["noise"], cfg["n_coarse"], cfg["n_fine"],
                           cfg["n_fine_depth"], 0.01, fpc.case_composite(case), stage=False)
    print(f"{case['name']}: {res}")
    return res["moved"]


def _emulated_training_step(case, gt, backward=True):
    """pnr_render then pnr_render_backward on the emulator for loss = MSE(coarse) + MSE(fine) (train.py:199-212)."""
    pn = eu.pn
    cfg = case["cfg"]
    keep = []
    scene = eu.scene_struct(case, gu.oracle_state(case), keep)
    mc = eu.mlp_struct(case["wc"], cfg["d_hidden"])
    mf = eu.mlp_struct(case["wf"], cfg["d_hidden"]) if case["wf"] is not None else None
    R, Kc, Kf, Kfd = cfg["SB"] * cfg["B"], cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"]
    rc = pn.PnrRenderCfg()
    rc.n_coarse, rc.n_fine, rc.n_fine_depth, rc.depth_std = Kc, Kf, Kfd, 0.01
    rc.white_bkgd, rc.engine = int(bool(cfg["white_bkgd"])), 1
    nz = {k: v.contiguous() for k, v in case["noise"].items()}
    lin = torch.linspace(0, 1 - 1.0 / Kc, Kc)
    noise = pn.PnrNoise()
    noise.lin_steps, noise.u_coarse = eu.ptr(lin), eu.ptr(nz["u_coarse"])
    if Kf - Kfd > 0:
        noise.u_fine, noise.u_fine_jit = eu.ptr(nz["u_fine"]), eu.ptr(nz["u_fine_jit"])
    if Kfd > 0:
        noise.n_depth = eu.ptr(nz["n_depth"])
    t = dict(rgb_coarse=torch.empty(R, 3), depth_coarse=torch.empty(R), weights_coarse=torch.empty(R, Kc),
             z_coarse=torch.empty(R, Kc))
    if Kf > 0:
        t.update(rgb_fine=torch.empty(R, 3), depth_fine=torch.empty(R), weights_fine=torch.empty(R, Kc + Kf),
                 z_fine=torch.empty(R, Kc + Kf))
    o = pn.PnrRenderOut()
    for k, v in t.items():
        setattr(o, k, eu.ptr(v))
    rays = case["rays"].contiguous()
    L = eu.lib()
    nbytes = L.pnr_render_workspace_bytes(scene, mc, mf, rc, cfg["B"])
    ws = torch.empty(nbytes, dtype=torch.uint8)
    eu.ok(L.pnr_render(scene, mc, mf, rc, eu.ptr(rays), noise, o, cfg["B"], ws.data_ptr(), nbytes, None))
    if not backward:
        return None, None, None, None, t
    gtf = gt.reshape(-1, 3)
    loss = torch.nn.functional.mse_loss(t["rgb_coarse"], gtf)
    d_c = (2.0 * (t["rgb_coarse"] - gtf) / gtf.numel()).contiguous()
    d_f = None
    if Kf > 0:
        loss = loss + torch.nn.functional.mse_loss(t["rgb_fine"], gtf)
        d_f = (2.0 * (t["rgb_fine"] - gtf) / gtf.numel()).contiguous()
    g_c = {k: torch.zeros_like(v) for k, v in case["wc"].items()}
    g_f = {k: torch.zeros_like(v) for k, v in case["wf"].items()} if case["wf"] is not None else None
    gsc = eu.mlp_struct(g_c, cfg["d_hidden"])
    gsf = eu.mlp_struct(g_f, cfg["d_hidden"]) if g_f is not None else None
    V, Cc, Hl, Wl = case["latent"].shape
    d_lat = torch.zeros(V, Hl, Wl, Cc)
    nbytes = L.pnr_render_backward_workspace_bytes(scene, mc, mf, rc, cfg["B"])
    ws = torch.empty(nbytes, dtype=torch.uint8)
    eu.ok(L.pnr_render_backward(scene, mc, mf, rc, eu.ptr(rays), noise, o, eu.ptr(d_c), eu.ptr(d_f), gsc, gsf,
                                eu.ptr(d_lat), cfg["B"], ws.data_ptr(), nbytes, None))
    return loss.item(), g_c, g_f, d_lat.permute(0, 3, 1, 2), t


@pytest.mark.parametrize("name", gu.GRAD_CASE_NAMES + ["ns1_coarse_only"])
def test_emulated_training_step_gradients(name):
    """The whole backward of a training step through the C ABI (CUDA sources on the host emulator) against
    (a) the hand-derived oracle backward and (b), where a fixture exists, the gradients the reference produced."""
    case = gu.load_case(name)
    cfg = case["cfg"]
    has_fixture = name in gu.GRAD_CASE_NAMES
    gt = gu.load_grad_case(name)["rgb_gt"] if has_fixture else torch.rand(
        cfg["SB"], cfg["B"], 3, generator=torch.Generator().manual_seed(1))
    loss, g_c, g_f, d_lat, fwd = _emulated_training_step(case, gt)
    m_loss, o_c, o_f, o_lat = bw.train_loss_backward(case["rays"], gt, case["noise"], gu.oracle_state(case),
                                                     case["latent"], case["wc"], case["wf"], cfg["NS"],
                                                     cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"],
                                                     white_bkgd=bool(cfg["white_bkgd"]))
    if cfg["n_fine"] > 0:    # the comparison needs identical samples: no ray may have flipped a CDF bin
        ref = gu.oracle_render(case)
        assert (fwd["z_fine"] - ref["fine"]["z"]).abs().max() < 1e-5
    assert abs(loss - m_loss.item()) < 1e-5
    assert rel(d_lat, o_lat) < 2e-4
    for k in o_c:
        assert rel(g_c[k], o_c[k]) < 2e-4, ("coarse", k)
    if o_f is not None:
        for k in o_f:
            assert rel(g_f[k], o_f[k]) < 2e-4, ("fine", k)
    if has_fixture:
        g = gu.load_grad_case(name)
        assert abs(loss - g["loss"]) < 1e-5
        assert rel(d_lat, g["g_latent"]) < 5e-4
        for k, v in g["gc"].items():
            assert rel(g_c[k], v) < 5e-4, ("coarse vs reference", k)
        for k, v in g["gf"].items():
            assert rel(g_f[k], v) < 5e-4, ("fine vs reference", k)


def test_emulated_caller_side_and_layout_kernels():
    """k_gen_rays (warp shuffles), k_frames_u8, k_pack_latent (shared-memory transpose) on the emulator against the
    reference-generated fixtures / plain torch."""
    import numpy as np
    L = eu.lib()
    z = np.load(gu.GOLD + "/util_rays.npz")
    poses = torch.from_numpy(z["poses"]).contiguous()
    for first, count in ((0, 3 * 9 * 12), (7, 100), (300, 24)):
        rays = torch.empty(count, 8)
        eu.ok(L.pnr_gen_rays(eu.ptr(poses), 3, 12, 9, 13.5, 13.5, 6.0, 4.5, 0.8, 1.8, first, count, eu.ptr(rays), None))
        want = torch.from_numpy(z["rays"]).reshape(-1, 8)[first:first + count]
        assert (rays - want).abs().max() < 1e-6
    f = np.load(gu.GOLD + "/frames_u8.npz")
    rgb = torch.from_numpy(f["rgb"]).contiguous()
    out = torch.empty(rgb.shape, dtype=torch.uint8)
    eu.ok(L.pnr_frames_u8(eu.ptr(rgb), rgb.numel(), out.data_ptr(), None))
    assert np.array_equal(out.numpy(), f["u8"])
    lat = torch.randn(2, 48, 5, 7, generator=torch.Generator().manual_seed(1))
    nhwc = torch.empty(2, 5, 7, 48)
    eu.ok(L.pnr_pack_latent(eu.ptr(lat), eu.ptr(nhwc), 2, 48, 5, 7, None))
    assert torch.equal(nhwc, lat.permute(0, 2, 3, 1).contiguous())


@pytest.mark.parametrize("n_fine,n_fine_depth", [(6, 0), (4, 4), (5, 1)])
def test_emulated_training_step_sample_count_edge_cases(n_fine, n_fine_depth):
    """No depth-centred samples (no position gradient needed), only depth-centred samples (no importance samples),
    and a single one -- against the hand-derived oracle backward with the same noise."""
    import copy
    case = copy.copy(gu.load_case("sb2_d"))
    cfg = dict(case["cfg"], n_fine=n_fine, n_fine_depth=n_fine_depth)
    case["cfg"] = cfg
    R = cfg["SB"] * cfg["B"]
    case["noise"] = gu.synth.draw_noise(77, R, cfg["n_coarse"], n_fine, n_fine_depth)
    gt = torch.rand(cfg["SB"], cfg["B"], 3, generator=torch.Generator().manual_seed(3))
    loss, g_c, g_f, d_lat, fwd = _emulated_training_step(case, gt)
    m_loss, o_c, o_f, o_lat = bw.train_loss_backward(case["rays"], gt, case["noise"], gu.oracle_state(case),
                                                     case["latent"], case["wc"], case["wf"], cfg["NS"],
                                                     cfg["n_coarse"], n_fine, n_fine_depth,
                                                     white_bkgd=bool(cfg["white_bkgd"]))
    ref = gu.oracle_render(case)
    assert (fwd["z_fine"] - ref["fine"]["z"]).abs().max() < 1e-5      # identical samples (no flipped bin)
    assert abs(loss - m_loss.item()) < 1e-5
    assert rel(d_lat, o_lat) < 2e-4
    for k in o_c:
        assert rel(g_c[k], o_c[k]) < 2e-4, ("coarse", k)
    for k in o_f:
        assert rel(g_f[k], o_f[k]) < 2e-4, ("fine", k)
