"""The single-pass tensor engine (engine "tc_fast", PNR_ENGINE_TC_FAST) on the H100: against its CPU restatement
(tests/tc_fast_oracle.py) at a tight bound, against the fp32 oracle at the documented loose bound, at the true C2 / C3 /
C4 shapes, through bind_parallel and util.recon, and its refusals (grad mode, the backward entry points, shapes the
tensor engine cannot run).  The fine pass is checked on every ray against references conditioned on the kernel's own
coarse pass (tests/fine_pass_check.py)."""
import ctypes as C
import importlib.util
import os

import numpy as np
import pytest
import torch

import fine_pass_check as fpc
import golden_util as gu
import gpu_util
import tc_fast_oracle as fo

pytestmark = pytest.mark.gpu

CASES = ["c2_small", "c3_small", "c4_small"]     # the d_hidden = 512 golden cases
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PNR_ERR_INVALID = -1              # include/pnr.h

# The bench.py parity block of the single-pass engine against the fp32 oracle (256 rays of a true-shape frame).
# Measured on an H100 (C2 / C3 / C4): max |d rgb| 1.9e-4 / 2.7e-4 / 2.8e-4 on rays that kept their bins (coarse pass
# up to 4.9e-4), p99.9 up to 2.8e-4, PSNR 85 / 70 / 69 dB, 16 / 35 / 113 flipped rays.
PARITY_MAX_DRGB = 2e-3
PARITY_P999_DRGB = 2e-3
PARITY_PSNR_DB = 55.0
RECON_SIGMA = 5e-3                # util.recon sigma grid: max |d sigma| / (1 + max |sigma|); measured 5.2e-4


def _cpu(res):
    return {p: {k: v.cpu() for k, v in d.items()} for p, d in res.items()}


@pytest.mark.parametrize("name", CASES)
def test_render_against_restatement_and_oracle(name):
    import pnr_native as pn
    case = gu.load_case(name)
    res = _cpu(gpu_util.render_case_cuda(case, engine="tc_fast"))
    assert pn.tc_status() == 0
    tight = fo.render_errors(res, fo.render(case))
    ref = gu.oracle_render(case)
    loose = fo.render_errors(res, ref)
    print(f"{name}: vs restatement {tight}  vs fp32 oracle {loose}")
    assert (res["coarse"]["z"] - ref["coarse"]["z"]).abs().max() < 1e-6      # the stratified samples are exact
    assert tight["coarse"] < fo.TIGHT_RGB, tight
    assert loose["coarse"] < fo.LOOSE_RGB, loose
    # every ray's fine pass at the kernel's own samples: against the restatement and against the fp32 oracle
    chk = fpc.check_case(case, res, arithmetic=fo.arithmetic, rgb_tol=fo.TIGHT_RGB, depth_tol=None, weights_tol=None)
    chk_loose = fpc.check_fine_outputs(case["rays"], res["fine"]["z"], res["fine"], fpc.case_composite(case),
                                       rgb_tol=fo.LOOSE_RGB, depth_tol=None, weights_tol=None)
    print(f"{name} tc_fast: vs restatement {chk}  vs fp32 oracle {chk_loose}")


@pytest.mark.parametrize("name", CASES)
def test_field_against_restatement_and_oracle(name):
    """PixelNeRFNet.forward (pnr_field_eval) on the golden cases' scattered points (incl. behind-camera / off-image)."""
    case = gu.load_case(name)
    net = gpu_util.build_net(case, engine="tc_fast")
    r = case["ref"]
    for coarse, key in ((True, "field_coarse"), (False, "field_fine")):
        with torch.no_grad():
            out = net(r["field_xyz"].cuda(), coarse=coarse, viewdirs=r["field_dirs"].cuda()).cpu()
        fast = fo.field(case, r["field_xyz"], r["field_dirs"], coarse=coarse)
        tight = ((out - fast).abs() / (1 + fast.abs())).max().item()
        loose = ((out - r[key]).abs() / (1 + r[key].abs())).max().item()
        print(f"{name} {key}: vs restatement {tight:.2e}  vs fp32 oracle {loose:.2e}")
        assert tight < fo.TIGHT_FIELD, (key, tight)
        assert loose < fo.LOOSE_FIELD, (key, loose)


def test_unsupported_shape_is_refused():
    """sb2_d is 32 wide: the single-pass engine, like "tc", refuses it instead of falling back to the SIMT engine."""
    case = gu.load_case("sb2_d")
    assert case["cfg"]["d_hidden"] != 512
    with pytest.raises(RuntimeError, match="PNR_ENGINE_TC_FAST"):
        gpu_util.render_case_cuda(case, engine="tc_fast")
    net = gpu_util.build_net(case, engine="tc_fast")
    with torch.no_grad(), pytest.raises(RuntimeError, match="PNR_ENGINE_TC_FAST"):
        net(case["ref"]["field_xyz"].cuda(), coarse=True, viewdirs=case["ref"]["field_dirs"].cuda())


def test_two_runs_bit_identical_and_auto_is_tc():
    case = gu.load_case("c2_small")
    a, b = (_cpu(gpu_util.render_case_cuda(case, engine="tc_fast")) for _ in range(2))
    tc, auto = (_cpu(gpu_util.render_case_cuda(case, engine=e)) for e in ("tc", "auto"))
    for p in ("coarse", "fine"):
        for k in a[p]:
            assert torch.equal(a[p][k], b[p][k]), (p, k)
            assert torch.equal(auto[p][k], tc[p][k]), (p, k)
    assert not torch.equal(a["fine"]["rgb"], tc["fine"]["rgb"])     # the single pass really ran


def _load_bench():
    spec = importlib.util.spec_from_file_location("pnr_bench", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("name", ["c2", "c3", "c4"])
def test_parity_block_at_true_shapes(name):
    """bench.py's parity block (256 rays spread over a true-shape frame, injected noise, CPU fp32 oracle) with the
    single-pass engine."""
    import pnr_native as pn
    bench = _load_bench()
    cfg = bench.synth.CONFIGS[name]
    net, renderer = bench.build_scene(cfg, torch.device("cuda:0"), "tc_fast")
    rays = bench.synth.make_rays(cfg, bench.WORKLOADS[name]["frame_rays"]).cuda()[None]
    par = bench.parity_block(net, renderer, cfg, rays, n=256)
    assert pn.tc_status() == 0
    print(f"{name} tc_fast parity: " + ", ".join(f"{k}={par[k]}" for k in (
        "psnr_db", "max_abs_drgb_coarse", "max_abs_drgb", "p999_abs_drgb", "max_abs_drgb_incl_flipped",
        "flipped_rays")))
    assert par["rays"] == 256
    assert par["max_abs_drgb_coarse"] < PARITY_MAX_DRGB, par
    assert par["max_abs_drgb"] < PARITY_MAX_DRGB, par
    assert par["p999_abs_drgb"] < PARITY_P999_DRGB, par
    assert par["psnr_db"] > PARITY_PSNR_DB, par
    # the same rays and noise, every ray's fine pass checked; the float64 restatement on a fixed subset of them
    chk = fpc.check_true_shape(bench, net, renderer, cfg, rays, n=256, arithmetic=fo.arithmetic, n_sub=96,
                               rgb_tol=fo.TIGHT_RGB, depth_tol=None, weights_tol=None)
    assert pn.tc_status() == 0
    print(f"{name} tc_fast: vs restatement {chk}")


def test_bind_parallel_two_shards_bit_equal_to_one_gpu():
    """bind_parallel(net, [0, 0]) runs pnr_mgpu_render with two shards on one device; cfg.engine reaches every shard.
    Shard i draws its noise from the device's generator after shard i-1, so rendering the two ray ranges one after
    the other on one GPU from the same seed gives the same draws."""
    bench = _load_bench()
    cfg = bench.synth.CONFIGS["c2"]
    net, renderer = bench.build_scene(cfg, torch.device("cuda:0"), "tc_fast")
    n = 1001
    rays = bench.synth.make_rays(cfg, n).cuda()[None]
    par = renderer.bind_parallel(net, [0, 0], simple_output=True).eval()
    one = renderer.bind_parallel(net, [0], simple_output=True).eval()
    k = -(-n // 2)
    with torch.no_grad():
        torch.manual_seed(3)
        rgb, depth = par(rays)
        torch.manual_seed(3)
        a, b = one(rays[:, :k]), one(rays[:, k:])
        net.engine = "tc"
        torch.manual_seed(3)
        exact = torch.cat((one(rays[:, :k])[0], one(rays[:, k:])[0]), dim=1)
    assert torch.equal(rgb, torch.cat((a[0], b[0]), dim=1))
    assert torch.equal(depth, torch.cat((a[1], b[1]), dim=1))
    assert not torch.equal(rgb, exact)             # the shards ran the single-pass engine


def test_recon_marching_cubes_on_c2_scene(monkeypatch):
    """util.recon.marching_cubes with the single-pass engine: sigma against the fp32 oracle and the restatement, the
    mesh is the oracle's marching cubes of the same volume, and the surface of that volume is closed."""
    from recon_util import recon
    from test_gpu_recon import C1_, C2_, RESO, _Spy, assert_same_mesh, c2_net
    from util import recon as urecon
    import pnr_native as pn
    net, state, latent = c2_net("tc_fast")
    spy = _Spy(monkeypatch)
    urecon.marching_cubes(net, C1_, C2_, [12, 12, 12], isosurface=1e9)
    iso = float(np.median(spy.vols[-1]))
    verts, tris = urecon.marching_cubes(net, C1_, C2_, RESO, isosurface=iso, eval_batch_size=20000)
    vol = spy.vols[-1]
    pts = recon.grid_points(C1_, C2_, RESO)
    idx = np.linspace(0, len(pts) - 1, 1500).astype(np.int64)
    p = torch.from_numpy(pts[idx])[None]
    d = torch.from_numpy(recon.fake_viewdirs(pts[idx]))[None]
    w = gu.synth.bench_mlp_weights(11, 512)
    got = vol.reshape(-1)[idx]
    ref = gu.oracle.field_eval(p, d, state, latent, w, 2)[0, :, 3].numpy()
    fast = fo.field_eval(p, d, state, latent, w, 2)[0, :, 3].numpy()
    scale = 1.0 + np.abs(ref).max()
    err, tight = float(np.abs(got - ref).max() / scale), float(np.abs(got - fast).max() / scale)
    print(f"recon sigma: vs fp32 oracle {err:.2e}, vs restatement {tight:.2e}")
    assert err <= RECON_SIGMA and tight <= fo.TIGHT_FIELD
    rv, rt = recon.marching_cubes(vol, iso)
    rv = rv * ((np.array(C2_) - np.array(C1_)) / np.array(RESO)) + np.array(C1_)
    assert len(rt) > 1000
    assert_same_mesh(verts, tris, rv, rt)
    # padded with an outside border the extracted surface is closed and consistently oriented (watertight)
    padded = np.pad(vol, 1, constant_values=np.float32(iso - 1.0))
    _, pt = pn.marching_cubes(torch.from_numpy(padded).cuda(), iso)
    assert recon.is_closed_oriented(pt.cpu().numpy())


def test_grad_mode_is_refused_by_name():
    case = gu.load_case("c2_small")
    net = gpu_util.build_net(case, engine="tc_fast")
    renderer = gpu_util.build_renderer(case)
    rays = case["rays"].cuda()
    r = case["ref"]
    assert any(p.requires_grad for p in net.mlp_coarse.parameters())
    with pytest.raises(RuntimeError, match='"tc_fast".*"tc" or "auto"'):
        renderer(net, rays)                                                  # fused_render_train
    with pytest.raises(RuntimeError, match='"tc_fast".*"tc" or "auto"'):
        net(r["field_xyz"].cuda(), coarse=True, viewdirs=r["field_dirs"].cuda())   # fused_field
    with pytest.raises(RuntimeError, match='"tc_fast".*"tc" or "auto"'):
        renderer.bind_parallel(net, [0, 0])(rays)                           # _ShardedFusedRender
    with torch.no_grad():
        renderer(net, rays)                                                  # inference is fine
    net.engine = "tc"
    out = renderer(net, rays)
    out.fine.rgb.sum().backward()                                            # training with "tc" still runs
    assert net.mlp_coarse.lin_out.weight.grad is not None


def test_backward_entry_points_refuse_the_engine():
    """The C ABI refuses PNR_ENGINE_TC_FAST in the render backward entry points (single and multi-GPU) with
    PNR_ERR_INVALID instead of differentiating the exact engine's forward."""
    import pnr_native as pn
    case = gu.load_case("c2_small")
    net = gpu_util.build_net(case, engine="tc")
    cfg_c = case["cfg"]
    scene, mc, mf, keep = net._scene_struct(want_fine=True)
    cfg = pn.PnrRenderCfg(cfg_c["n_coarse"], cfg_c["n_fine"], cfg_c["n_fine_depth"], 0.01, 1, pn.ENGINE_TC_FAST)
    noise, fwd, up = pn.PnrNoise(), pn.PnrRenderOut(), pn.PnrRenderGrad()
    L = pn.lib()
    B = case["rays"].shape[1]
    rc = L.pnr_render_backward_ex(scene, mc, mf, cfg, None, noise, fwd, up, mc, mf, None, B, None, 0, None)
    assert rc == PNR_ERR_INVALID and b"PNR_ENGINE_TC_FAST" in L.pnr_last_error()
    rc = L.pnr_render_backward(scene, mc, mf, cfg, None, noise, fwd, None, None, mc, mf, None, B, None, 0, None)
    assert rc == PNR_ERR_INVALID and b"PNR_ENGINE_TC_FAST" in L.pnr_last_error()
    rc = L.pnr_render_backward_cam(scene, mc, mf, cfg, None, noise, fwd, up, mc, mf, None, None, None, B, None, 0,
                                   None)
    assert rc == PNR_ERR_INVALID and b"PNR_ENGINE_TC_FAST" in L.pnr_last_error()
    h = C.c_void_p()
    ids = (C.c_int32 * 2)(0, 0)
    pn.check(L.pnr_mgpu_create(ids, 2, C.byref(h)))
    try:
        shards, sgs = (pn.PnrShard * 2)(), (pn.PnrShardGrad * 2)()
        rc = L.pnr_mgpu_render_backward(h, shards, sgs, cfg, up, mc, mf, None, B, None)
        assert rc == PNR_ERR_INVALID and b"PNR_ENGINE_TC_FAST" in L.pnr_last_error()
    finally:
        L.pnr_mgpu_destroy(h)
    # the exact engine's workspace query answers for the fast engine too (the forward's)
    assert L.pnr_render_workspace_bytes(scene, mc, mf, cfg, B) == L.pnr_render_workspace_bytes(
        scene, mc, mf, pn.PnrRenderCfg(cfg_c["n_coarse"], cfg_c["n_fine"], cfg_c["n_fine_depth"], 0.01, 1,
                                       pn.ENGINE_TC), B)
