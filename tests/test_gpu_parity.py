"""GPU parity: the CUDA path (through the Python surface and the C ABI) against the CPU
oracle on the golden cases.  Tolerances: |d rgb| < 1e-4 (BASELINE.json north_star),
sample depths / weights 1e-5.  The fine pass is checked on every ray against a reference conditioned on the
kernel's own coarse pass (tests/fine_pass_check.py): an importance sample may take the bin next to the oracle's only
when its u lies within fp32 rounding of the cdf edge between them."""
import pytest
import torch

import fine_pass_check as fpc
import golden_util as gu

pytestmark = pytest.mark.gpu

# every golden case on the fp32 SIMT engine, and the d_hidden = 512 cases also on the tensor engine (the product
# default: engine "auto" picks it whenever the shape allows)
TC_CASES = ["c2_small", "c3_small", "c4_small"]
CASE_ENGINE = [(n, "simt") for n in gu.CASE_NAMES] + [(n, "tc") for n in TC_CASES] + [(n, "auto") for n in TC_CASES]


@pytest.mark.parametrize("name,engine", CASE_ENGINE)
def test_render_parity(name, engine):
    import gpu_util
    case = gu.load_case(name)
    res = gpu_util.render_case_cuda(case, engine=engine)
    ref = gu.oracle_render(case)
    c, rc = res["coarse"], ref["coarse"]
    assert (c["z"].cpu() - rc["z"]).abs().max() < 1e-6
    assert (c["rgb"].cpu() - rc["rgb"]).abs().max() < 1e-4
    assert (c["depth"].cpu() - rc["depth"]).abs().max() < 1e-4
    assert (c["weights"].cpu() - rc["weights"]).abs().max() < 1e-4
    if case["cfg"]["n_fine"] > 0:
        chk = fpc.check_case(case, res)
        flipped = int(((res["fine"]["z"].cpu() - ref["fine"]["z"]).abs() > 2e-4).any(-1).sum())
        print(f"{name} {engine}: {chk}, {flipped} rays merged other samples than the oracle")


@pytest.mark.parametrize("name,engine", CASE_ENGINE)
def test_field_parity(name, engine):
    """PixelNeRFNet.forward on scattered points (incl. behind-camera / off-image)."""
    import gpu_util
    case = gu.load_case(name)
    net = gpu_util.build_net(case, engine=engine)
    ref = case["ref"]
    with torch.no_grad():
        out_c = net(ref["field_xyz"].cuda(), coarse=True, viewdirs=ref["field_dirs"].cuda())
        out_f = net(ref["field_xyz"].cuda(), coarse=False, viewdirs=ref["field_dirs"].cuda())
    for out, key in ((out_c, "field_coarse"), (out_f, "field_fine")):
        err = (out.cpu() - ref[key]).abs() / (1.0 + ref[key].abs())
        # fp32 engine: 5e-5 on everything; tensor engine: RGB (the contract, 1e-4 absolute) and sigma relative
        assert err.max() < (5e-5 if engine == "simt" else 5e-4), (key, err.max())
        assert (out.cpu()[..., :3] - ref[key][..., :3]).abs().max() < 1e-4


def test_stage_entry_points():
    """pnr_sample_coarse / pnr_composite / pnr_sample_fine individually vs the oracle."""
    import gpu_util  # noqa: F401  (sys.path)
    import pnr_native as pn
    case = gu.load_case("c2_small")
    cfg = case["cfg"]
    ref = gu.oracle_render(case)
    dev = torch.device("cuda:0")
    rays = case["rays"].reshape(-1, 8).to(dev).contiguous()
    R, Kc, Kf, Kfd = rays.shape[0], cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"]
    L = pn.lib()
    sp = pn.stream_ptr(dev)
    d = lambda t: t.to(dev).contiguous()  # keep every device tensor alive until the sync below
    n = case["noise"]
    u_c, zc_ref, wc_ref, dc_ref = d(n["u_coarse"]), d(ref["coarse"]["z"]), d(ref["coarse"]["weights"]), d(ref["coarse"]["depth"])
    u_f, u_j, n_d = d(n["u_fine"]), d(n["u_fine_jit"]), d(n["n_depth"])
    z = torch.empty(R, Kc, device=dev)
    pn.check(L.pnr_sample_coarse(pn.dptr(rays), None, pn.dptr(u_c), pn.dptr(z), R, Kc, sp))
    assert (z.cpu() - ref["coarse"]["z"]).abs().max() < 1e-6
    # composite on the oracle's field values
    st = gu.oracle_state(case)
    r8 = case["rays"].reshape(-1, 8)
    pts = r8[:, None, :3] + ref["coarse"]["z"].unsqueeze(2) * r8[:, None, 3:6]
    dirs = r8[:, None, 3:6].expand(-1, Kc, -1)
    field = gu.oracle.field_eval(pts.reshape(1, -1, 3), dirs.reshape(1, -1, 3), st, case["latent"], case["wc"], cfg["NS"])
    field = d(field.reshape(R, Kc, 4))
    w = torch.empty(R, Kc, device=dev); rgb = torch.empty(R, 3, device=dev); dep = torch.empty(R, device=dev)
    pn.check(L.pnr_composite(pn.dptr(rays), pn.dptr(zc_ref), pn.dptr(field), 1, pn.dptr(w), pn.dptr(rgb), pn.dptr(dep), R, Kc, sp))
    assert (w.cpu() - ref["coarse"]["weights"]).abs().max() < 1e-6
    assert (rgb.cpu() - ref["coarse"]["rgb"]).abs().max() < 1e-5
    zf = torch.empty(R, Kc + Kf, device=dev)
    pn.check(L.pnr_sample_fine(pn.dptr(rays), pn.dptr(zc_ref), pn.dptr(wc_ref), pn.dptr(dc_ref), pn.dptr(u_f), pn.dptr(u_j),
                               pn.dptr(n_d), 0.01, pn.dptr(zf), R, Kc, Kf, Kfd, sp))
    torch.cuda.synchronize()
    # the oracle's coarse pass as input: every ray's merge explained against the float64 cdf of those weights
    moved = fpc.explain_fine_z(rays, zc_ref, wc_ref, dc_ref, n, Kc, Kf, Kfd, 0.01, zf)
    print(f"pnr_sample_fine on the oracle's coarse pass: {moved} importance samples in a non-float64 bin")


@pytest.mark.parametrize("name,engine", [("tiny", "simt"), ("c2_small", "auto")])
def test_public_api_seeded_and_empty(name, engine):
    """NeRFRenderer.forward / bind_parallel surface: shapes, determinism under a seed, empty shard."""
    import gpu_util
    case = gu.load_case(name)
    net = gpu_util.build_net(case, engine=engine)
    renderer = gpu_util.build_renderer(case)
    rays = case["rays"].cuda()
    par = renderer.bind_parallel(net, [0], simple_output=True).eval()
    with torch.no_grad():
        torch.manual_seed(7); rgb1, d1 = par(rays)
        torch.manual_seed(7); rgb2, d2 = par(rays)
        full = renderer.bind_parallel(net, None, simple_output=False)(rays, want_weights=True)
        e_rgb, e_d = par(rays[:0])
    assert rgb1.shape == (1, rays.shape[1], 3) and d1.shape == (1, rays.shape[1])
    assert torch.equal(rgb1, rgb2) and torch.equal(d1, d2)
    assert set(full.keys()) == {"coarse", "fine"} and "weights" in full["fine"]
    assert e_rgb.shape[0] == 0


def test_no_cpu_fallback():
    import gpu_util
    case = gu.load_case("tiny")
    net = gpu_util.build_net(case, device="cpu", engine="simt")
    with torch.no_grad(), pytest.raises(RuntimeError):
        net(case["ref"]["field_xyz"], coarse=True, viewdirs=case["ref"]["field_dirs"])


@pytest.mark.parametrize("name,engine", [("tiny", "simt"), ("c2_small", "tc")])
@pytest.mark.parametrize("n_fine,n_fine_depth", [(6, 0), (5, 5), (0, 0)])
def test_sample_count_edge_cases(n_fine, n_fine_depth, name, engine):
    """No depth samples / no importance samples / coarse only (nerf.py:284-293 skips the empty sampler)."""
    import gpu_util
    case = gu.load_case(name)
    cfg = dict(case["cfg"])
    cfg.update(n_fine=n_fine, n_fine_depth=n_fine_depth)
    case = dict(case, cfg=cfg)
    R = case["rays"].shape[0] * case["rays"].shape[1]
    case["noise"] = gu.synth.draw_noise(77, R, cfg["n_coarse"], n_fine, n_fine_depth)
    res = gpu_util.render_case_cuda(case, engine=engine)
    ref = gu.oracle_render(case)
    assert (res["coarse"]["rgb"].cpu() - ref["coarse"]["rgb"]).abs().max() < 1e-4
    if n_fine > 0:
        chk = fpc.check_case(case, res, depth_tol=2e-4)
        print(f"{name} {engine} ({n_fine}, {n_fine_depth}): {chk}")
    else:
        assert "fine" not in res
