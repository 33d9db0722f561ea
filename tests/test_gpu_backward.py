"""pnr_field_backward / pnr_render_backward (fp32 SIMT recompute-in-backward; the default training path on CUDA) against
the gradients the reference produced itself (tests/golden/grad_*.npz), the oracle's hand-written backward formulas
and the composed-torch grad-mode path."""
import os

import pytest
import torch

import golden_util as gu

pytestmark = pytest.mark.gpu


def rel(a, ref):
    return ((a - ref).abs().max() / (ref.abs().max() + 1e-20)).item()


def training_step(case, gt, fused):
    """fused: False = composed torch, 1 = field-level node (pnr_field_backward), 2 = render-level node
    (pnr_render + pnr_render_backward)."""
    import gpu_util
    os.environ["PNR_FUSED_BACKWARD"] = str(int(fused)) if fused != "auto" else "auto"
    net = gpu_util.build_net(case, device="cuda:0", engine="simt").train()
    net.encoder.latent = case["latent"].cuda().clone().requires_grad_(True)
    renderer = gpu_util.build_renderer(case).train()
    render_par = renderer.bind_parallel(net, None).train()
    torch.manual_seed(case["seed"] + 4)
    out = render_par(case["rays"].cuda(), want_weights=True)
    crit = torch.nn.MSELoss()
    loss = crit(out["coarse"]["rgb"], gt.cuda())
    if case["cfg"]["n_fine"] > 0:
        loss = loss + crit(out["fine"]["rgb"], gt.cuda())
    loss.backward()
    return loss.item(), net


@pytest.mark.parametrize("mode", [1, 2, "auto"])
@pytest.mark.parametrize("name", gu.GRAD_CASE_NAMES)
def test_fused_backward_matches_composed_torch_on_the_same_device(name, mode):
    """Same device RNG for both runs, so the samples are identical and only the backward differs."""
    case, g = gu.load_case(name), gu.load_grad_case(name)
    try:
        l0, ref = training_step(case, g["rgb_gt"], fused=False)
        l1, net = training_step(case, g["rgb_gt"], fused=mode)
    finally:
        os.environ.pop("PNR_FUSED_BACKWARD", None)
    assert abs(l0 - l1) < 1e-5
    assert rel(net.encoder.latent.grad, ref.encoder.latent.grad) < 1e-3
    for (k, p), (_, q) in zip(net.mlp_coarse.named_parameters(), ref.mlp_coarse.named_parameters()):
        assert rel(p.grad, q.grad) < 1e-3, ("coarse", k)
    if net.mlp_fine is not None:
        for (k, p), (_, q) in zip(net.mlp_fine.named_parameters(), ref.mlp_fine.named_parameters()):
            assert rel(p.grad, q.grad) < 1e-3, ("fine", k)


@pytest.mark.parametrize("name", gu.GRAD_CASE_NAMES)
def test_field_backward_matches_oracle_formulas(name):
    """Bare field: d_out random -> weight / latent / position gradients vs oracle/pnr_backward.py::field_backward."""
    import gpu_util
    bw = gu.load_by_path("pnr_backward", os.path.join(gu.ROOT, "oracle", "pnr_backward.py"))
    case = gu.load_case(name)
    cfg = case["cfg"]
    ref = case["ref"]
    xyz, dirs = ref["field_xyz"], ref["field_dirs"]
    g = torch.Generator().manual_seed(5)
    d_out = torch.randn(xyz.shape[0], xyz.shape[1], 4, generator=g)
    _, sv = bw.field_forward_saved(xyz, dirs, gu.oracle_state(case), case["latent"], case["wc"], cfg["NS"])
    g_ref, dlat_ref, dxyz_ref = bw.field_backward(sv, d_out)
    os.environ["PNR_FUSED_BACKWARD"] = "1"
    try:
        net = gpu_util.build_net(case, device="cuda:0", engine="simt").train()
        net.encoder.latent = case["latent"].cuda().clone().requires_grad_(True)
        x = xyz.cuda().clone().requires_grad_(True)
        out = net(x, coarse=True, viewdirs=dirs.cuda())
        out.backward(d_out.cuda())
    finally:
        os.environ.pop("PNR_FUSED_BACKWARD", None)
    assert rel(x.grad.cpu(), dxyz_ref) < 1e-3
    assert rel(net.encoder.latent.grad.cpu(), dlat_ref) < 1e-3
    for k, p in net.mlp_coarse.named_parameters():
        assert rel(p.grad.cpu(), g_ref[k]) < 1e-3, k


@pytest.mark.parametrize("name", gu.GRAD_CASE_NAMES)
def test_fused_training_step_matches_the_reference_gradients(name):
    """The default CUDA training path (pnr_render + pnr_render_backward in one autograd node) with the fixture's draws
    injected: loss and every gradient equal what the UNMODIFIED reference computed for train/train.py:199-215
    (tests/golden/grad_*.npz) to <= 1e-3 relative."""
    import gpu_util
    from render.fused_train import fused_render_train
    case, g = gu.load_case(name), gu.load_grad_case(name)
    net = gpu_util.build_net(case, device="cuda:0", engine="auto").train()
    net.encoder.latent = case["latent"].cuda().clone().requires_grad_(True)
    renderer = gpu_util.build_renderer(case).train()
    noise = {k: v.cuda() for k, v in case["noise"].items()}
    out = fused_render_train(renderer, net, case["rays"].cuda(), True, noise_in=noise)
    crit = torch.nn.MSELoss()
    gt = g["rgb_gt"].cuda()
    loss = crit(out.coarse.rgb, gt)
    if case["cfg"]["n_fine"] > 0:
        loss = loss + crit(out.fine.rgb, gt)
    assert abs(loss.item() - g["loss"]) < 1e-5
    loss.backward()
    assert rel(net.encoder.latent.grad.cpu(), g["g_latent"]) < 1e-3
    for k, p in net.mlp_coarse.named_parameters():
        assert rel(p.grad.cpu(), g["gc"][k]) < 1e-3, ("coarse", k)
    if net.mlp_fine is not None:
        for k, p in net.mlp_fine.named_parameters():
            assert rel(p.grad.cpu(), g["gf"][k]) < 1e-3, ("fine", k)


def test_gemm_nt_fp16_split_engine():
    """The projection's engine (fp16 hi/lo operands): latent-sized values times kaiming-sized weights, 22 mantissa bits."""
    import gpu_util  # noqa: F401
    import pnr_native as pn
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(3)
    M, N, K = 1000, 512, 512
    A = torch.clamp_min(torch.randn(M, K, generator=g) * 19 + 4, 0).to(dev)      # synth.make_latent statistics
    W = (torch.randn(N, K, generator=g) * 0.0625).to(dev)
    b = torch.randn(N, generator=g).to(dev)
    C = torch.zeros(M, N, device=dev)
    pn.check(pn.lib().pnr_gemm_nt(pn.dptr(A), K, pn.dptr(W), pn.dptr(b), pn.dptr(C), N, M, N, K, 0, 0, 3, pn.stream_ptr(dev)))
    torch.cuda.synchronize()
    ref = A.double() @ W.double().t() + b.double()
    scale = (A.double().abs() @ W.double().abs().t()).max()
    assert ((C.double() - ref).abs().max() / scale) < 2e-6


@pytest.mark.parametrize("engine", ["simt", "tc"])
@pytest.mark.parametrize("M,N,K,relu,accum", [(300, 512, 512, True, False),     # forward layer, ragged M
                                               (512, 512, 4000, False, True),    # weight gradient: K = rows, split-K
                                               (4, 512, 1008, False, True),      # lin_out weight gradient
                                               (1000, 48, 512, False, False),    # d_feat = dh W_in
                                               (777, 130, 48, False, True)])     # ragged N, one k-step
def test_gemm_nt_engines(M, N, K, relu, accum, engine):
    """pnr_gemm_nt (the contraction of the backward path) against a float64 product: the fp32 FFMA engine to fp32
    rounding, the split-bf16 wgmma engine to 16-bit-mantissa operands (<= 3e-5 of the row/column scale)."""
    import gpu_util  # noqa: F401
    import pnr_native as pn
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(M + N + K)
    A = (torch.randn(M, K, generator=g) * 3e-4).to(dev)          # gradient-sized values: no scaling may be needed
    W = torch.randn(N, K, generator=g).to(dev)
    b = torch.randn(N, generator=g).to(dev) * 1e-3
    C0 = torch.randn(M, N + 8, generator=g).to(dev) * 1e-3       # ldc > N: the pad columns must stay untouched
    C = C0.clone()
    pn.check(pn.lib().pnr_gemm_nt(pn.dptr(A), K, pn.dptr(W), pn.dptr(b), pn.dptr(C), N + 8, M, N, K, int(relu), int(accum),
                                  pn.ENGINES[engine], pn.stream_ptr(dev)))
    torch.cuda.synchronize()
    Ad = torch.relu(A.double()) if relu else A.double()
    ref = Ad @ W.double().t() + b.double() + (C0[:, :N].double() if accum else 0.0)
    scale = (Ad.abs() @ W.double().abs().t()).max()
    err = (C[:, :N].double() - ref).abs().max() / scale
    assert err < (2e-6 if engine == "simt" else 3e-5), err
    assert torch.equal(C[:, N:], C0[:, N:])
