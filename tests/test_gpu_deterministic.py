"""Deterministic mode on the H100: with torch.use_deterministic_algorithms(True) the fused training path gives the same
bits run to run (ordered split-K, fixed-point latent scatter, gather-form encoder upsample backward), and stays within
rounding of the default path."""
import os
import subprocess
import sys
import textwrap

import pytest
import torch

import aux_grad_util as au
import golden_util as gu

pytestmark = pytest.mark.gpu
rel = au.rel
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def deterministic():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _step(net, renderer, rays, noise, ups, par):
    from test_gpu_mgpu_train import _step as step
    rays.grad = None
    for t in (net.poses, net.focal, net.c):
        t.grad = None
    outs, grads = step(net, renderer, rays, noise, ups, par)
    for name, t in (("rays", rays), ("poses", net.poses), ("focal", net.focal), ("c", net.c)):
        grads[name] = t.grad.clone()
    return outs, grads


def _c2(engine):
    from test_gpu_aux_grad import _c2_train_scene
    from test_gpu_mgpu_train import _draws, _random_ups
    dev = torch.device("cuda:0")
    net, renderer, rays = _c2_train_scene(dev, engine)
    for t in (net.poses, net.focal, net.c):
        t.requires_grad_(True)
    rays.requires_grad_(True)
    SB, B = rays.shape[:2]
    Kc, Kf, Kfd = renderer.n_coarse, renderer.n_fine, renderer.n_fine_depth
    return net, renderer, rays, _draws(SB * B, Kc, Kf, Kfd, 7, dev), _random_ups(SB, B, Kc, Kc + Kf, 9, dev)


@pytest.mark.parametrize("engine", ["tc", "simt"])
@pytest.mark.parametrize("gpus", [None, [0, 0]], ids=["one_gpu", "bind_parallel_0_0"])
@pytest.mark.parametrize("chunk_rows", [None, "4096", "1000"], ids=["natural", "split_masked", "ragged"])
def test_backward_is_bit_repeatable_at_c2_train_shape(engine, gpus, chunk_rows, deterministic, monkeypatch):
    """Three flag-on backward passes on the same draws: every MLP gradient, the latent, the rays, poses, focal and c
    are bit-identical; they agree with the default path to rounding.  PNR_BWD_CHUNK_ROWS covers the split-K regimes:
    the natural 32768-row chunk (weight-gradient GEMMs split), 4096 rows (every masked dX GEMM split too) and ragged
    1000-row chunks."""
    if chunk_rows:
        monkeypatch.setenv("PNR_BWD_CHUNK_ROWS", chunk_rows)
    net, renderer, rays, noise, ups = _c2(engine)
    par = renderer.bind_parallel(net, gpus).train() if gpus else None
    runs = [_step(net, renderer, rays, noise, ups, par) for _ in range(3)]
    for outs, grads in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(outs, runs[0][0]))
        assert grads.keys() == runs[0][1].keys()
        for k in grads:
            assert torch.equal(grads[k], runs[0][1][k]), k
    torch.use_deterministic_algorithms(False)
    off = [_step(net, renderer, rays, noise, ups, par)[1] for _ in range(2)]
    err = {k: rel(runs[0][1][k], off[0][k]) for k in off[0]}
    err_off = {k: rel(off[1][k], off[0][k]) for k in off[0]}
    worst = max(err, key=err.get)
    print(f"\n{engine} {gpus} {chunk_rows}: flag on vs off, worst relative gap {err[worst]:.2e} ({worst}), "
          f"latent {err['latent']:.2e}; two flag-off runs: {max(err_off.values()):.2e}")
    # At the natural chunk the recomputed forward's GEMMs do not split, so both modes see the same activations and
    # differ by summation order only.  With smaller chunks the recompute's GEMMs split too and the two modes associate
    # their sums differently (C + (P0 + P1) against (C + P0) + P1), which flips ReLU masks at width 512: measured
    # 1.5e-2 at 4096 rows, and 5e-6 with PNR_BWD_RECOMPUTE=simt, the same as two flag-off runs.  The bound there is
    # the one of the 512-wide tests that keep every point.
    assert err[worst] < (1e-4 if chunk_rows is None else 5e-2), sorted(err.items(), key=lambda kv: -kv[1])[:5]


def test_projection_and_render_are_bit_repeatable_on_a_c3_size_map(deterministic):
    """pnr_project_latent on a 1 x 512 x 32 x 32 map (its GEMM splits K) and a full render: the same bits three
    times; the projection cache keys on the flag, so turning it on re-projects."""
    import gpu_util
    case = gu.load_case("c3_small")
    net = gpu_util.build_net(case, engine="tc")
    lat = gu.synth.make_latent(11, 1, 32, 32).cuda()
    cfg = case["cfg"]
    net.set_scene(lat, case["src_poses"][:1, :1].cuda(), case["focal"].cuda(), None, cfg["W"], cfg["H"])
    renderer = gpu_util.build_renderer(case)
    rays = case["rays"].cuda()
    noise = {k: v.cuda() for k, v in case["noise"].items()}
    projs, outs = [], []
    for _ in range(3):
        net._fused.proj.clear()
        with torch.no_grad():
            scene, mc, mf, keep = net._scene_struct(want_fine=True)
            projs.append(keep[1]["mlp_coarse"].clone())
            o = renderer._forward_fused(net, rays, want_weights=True, noise_in=noise, want_z=True)
        outs.append(o["coarse"]["rgb"].clone())
    assert all(torch.equal(p, projs[0]) for p in projs[1:])
    assert all(torch.equal(o, outs[0]) for o in outs[1:])
    key_on = net._fused.proj["mlp_coarse"][0]
    torch.use_deterministic_algorithms(False)
    with torch.no_grad():
        net._scene_struct(want_fine=True)
    assert net._fused.proj["mlp_coarse"][0] != key_on
    assert rel(net._fused.proj["mlp_coarse"][1], projs[0]) < 1e-6


CHILD = textwrap.dedent("""
    import os, sys, hashlib
    os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
    import torch
    torch.use_deterministic_algorithms(True)
    torch.backends.cudnn.benchmark = False
    sys.path[:0] = [{tests!r}, {src!r}]
    import golden_util as gu, gpu_util
    from model import make_model
    from render import NeRFRenderer
    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    c2 = gu.synth.CONFIGS["c2"]
    SB, NS, B = 4, c2["NS"], 128
    net = make_model(gpu_util.model_conf(512)).to(dev).train()
    renderer = NeRFRenderer(n_coarse=c2["n_coarse"], n_fine=c2["n_fine"], n_fine_depth=c2["n_fine_depth"],
                            depth_std=0.01, white_bkgd=c2["white_bkgd"]).to(dev).train()
    par = renderer.bind_parallel(net, {gpus}).train()
    r = (c2["z_near"] + c2["z_far"]) * 0.5
    poses = torch.stack([torch.stack([gu.synth.pose_spherical(40.0 * v + 25.0 * o, -30.0, r) for v in range(NS)])
                         for o in range(SB)]).to(dev)
    g = torch.Generator().manual_seed(1)
    images = (torch.rand(SB, NS, 3, 128, 128, generator=g) * 2 - 1).to(dev)
    tgt = torch.stack([gu.synth.pose_spherical(100.0 + 70.0 * o, -10.0, r) for o in range(SB)])
    rays_all = gu.synth.gen_rays(tgt, c2["W"], c2["H"], c2["focal"], c2["z_near"], c2["z_far"]).reshape(SB, -1, 8)
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    losses = []
    for step in range(3):
        pix = torch.randint(0, rays_all.shape[1], (SB, B), generator=g)
        rays = torch.stack([rays_all[o][pix[o]] for o in range(SB)]).to(dev)
        gt = torch.rand(SB, B, 3, generator=g).to(dev)
        net.encode(images, poses, torch.tensor([c2["focal"]], device=dev))
        out = par(rays, want_weights=True)
        loss = ((out["coarse"]["rgb"] - gt) ** 2).mean() + ((out["fine"]["rgb"] - gt) ** 2).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    h = hashlib.sha256()
    for p in net.parameters():
        h.update(p.detach().cpu().numpy().tobytes())
    print("RESULT", [float.hex(x) for x in losses], h.hexdigest())
""")


@pytest.mark.parametrize("gpus", [[0], [0, 0]], ids=["one_gpu", "bind_parallel_0_0"])
def test_three_adam_steps_with_the_encoder_trained_are_bit_identical(gpus):
    """train.py's loss (encode with the encoder trained, render with want_weights, MSE coarse + fine) at SB = 4,
    B = 128 under torch.use_deterministic_algorithms(True): two runs from the same seed leave every parameter (encoder
    and both MLPs) and every loss bit-identical.  Without the deterministic upsample backward the encoder's
    F.interpolate backward raises here."""
    code = CHILD.format(tests=os.path.join(ROOT, "tests"), src=os.path.join(ROOT, "pixel-nerf_b200", "src"), gpus=gpus)
    res = []
    for _ in range(2):
        r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        res.append([l for l in r.stdout.splitlines() if l.startswith("RESULT")][-1])
    print("\n" + res[0])
    assert res[0] == res[1]


def _recording_rel(module, monkeypatch):
    """Wraps `module.rel` so that every relative error the module's test checks is also recorded -> the list."""
    seen = []
    inner = module.rel

    def rec(a, ref):
        e = float(inner(a, ref))
        seen.append(e)
        return e
    monkeypatch.setattr(module, "rel", rec)
    return seen


@pytest.mark.parametrize("name", gu.GRAD_CASE_NAMES)
def test_flag_on_training_step_matches_the_reference_gradients(name, deterministic, monkeypatch):
    """test_gpu_backward.py's comparison with the unmodified reference's gradients (tests/golden/grad_*.npz), its
    tolerances unchanged, with the flag on; prints the worst relative error."""
    import test_gpu_backward as tb
    seen = _recording_rel(tb, monkeypatch)
    tb.test_fused_training_step_matches_the_reference_gradients(name)
    print(f"\nflag on, {name}: worst relative error against the reference's gradients {max(seen):.2e}")


@pytest.mark.parametrize("engine", ["auto", "simt"])
@pytest.mark.parametrize("fixture", ["tiny", "sb2_d", "sb2_d_clamp"])
def test_flag_on_camera_gradients_match_the_reference(fixture, engine, deterministic, monkeypatch):
    """test_gpu_cam_grad.py's comparison with tests/golden/grad_cam_*.npz (rays, poses, focal, c, MLP), its tolerances
    unchanged, with the flag on; prints the worst relative error."""
    import test_gpu_cam_grad as tc
    seen = _recording_rel(tc, monkeypatch)
    tc.test_fused_node_matches_the_reference_camera_gradients(fixture, engine)
    print(f"\nflag on, {fixture} {engine}: worst relative error against the reference's gradients {max(seen):.2e}")


def test_flag_on_wide_backward_matches_float64_on_decided_points(deterministic):
    """test_gpu_backward_wide.py's cases with the flag on: the split-K, unsplit and ragged-chunk regimes of the
    512-wide backward against float64 on the decided points, within that file's TC_TOL with the default recompute and
    within its BWD_TOL with the forward recomputed on the fp32 SGEMM (a child interpreter: the library reads
    PNR_BWD_RECOMPUTE once per process).  This holds the ordered split-K sums of the masked, accumulating dX GEMMs and
    of the dW GEMMs to the tight bound."""
    import test_gpu_backward_wide as tw
    try:
        tw._check_cases(tw.CASES, tw.TC_TOL, "flag on")
    finally:
        os.environ.pop("PNR_BWD_CHUNK_ROWS", None)
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path.insert(0, {here!r}); import torch; "
            "torch.use_deterministic_algorithms(True, warn_only=True); import test_gpu_backward_wide as t; "
            "t._check_cases(t.CASES, t.BWD_TOL, 'flag on, fp32 recompute')")
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code],
                       env=dict(os.environ, PNR_BWD_RECOMPUTE="simt"), cwd=ROOT, capture_output=True, text=True)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-4000:]
