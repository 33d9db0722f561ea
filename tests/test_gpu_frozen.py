"""Training with part of the network frozen (render/fused_train.py -> pnr_render_backward_sel /
pnr_mgpu_render_backward_sel): under torch.use_deterministic_algorithms(True) every gradient a partly frozen step
computes is bit-equal to the same gradient of the step with everything trainable, on one GPU and through
bind_parallel(net, [0, 0]); frozen parameters keep .grad None.  With the flag off they agree within 1e-5 relative (the
weight-gradient GEMMs' split-K and the latent scatter then add with float atomics)."""
import warnings

import pytest
import torch

import aux_grad_util as au
import frozen_util as fu
import golden_util as gu

pytestmark = pytest.mark.gpu
rel = au.rel

CONFIGS = [("c2", "tc"), ("c2", "auto"), ("sb2_d", "auto"), ("tiny", "auto")]
_scenes, _full = {}, {}


def _scene(kind):
    if kind not in _scenes:
        _scenes[kind] = fu.Scene(kind, torch.device("cuda:0"))
    return _scenes[kind]


def _step(kind, engine, gpus, det, pattern):
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            res = _scene(kind).step(pattern, gpus, engine)
        assert not [w for w in caught if "bind_parallel" in str(w.message)], [str(w.message) for w in caught]
        return res
    finally:
        torch.use_deterministic_algorithms(prev)


def _full_step(kind, engine, gpus, det):
    key = (kind, engine, tuple(gpus or ()), det)
    if key not in _full:
        _full[key] = _step(kind, engine, gpus, det, fu.FULL)
    return _full[key]


@pytest.mark.parametrize("det", [True, False], ids=["deterministic", "flag_off"])
@pytest.mark.parametrize("gpus", [None, [0, 0]], ids=["one_gpu", "two_shards"])
@pytest.mark.parametrize("pattern", list(fu.PATTERNS))
@pytest.mark.parametrize("kind,engine", CONFIGS)
def test_frozen_step_gives_the_full_steps_gradients(kind, engine, pattern, gpus, det, monkeypatch):
    import pnr_native as pn
    L = pn.lib()
    sel_calls = []
    for name in ("pnr_render_backward_sel", "pnr_mgpu_render_backward_sel"):
        orig = getattr(L, name)
        monkeypatch.setattr(L, name, lambda *a, _o=orig, _n=name: sel_calls.append(_n) or _o(*a))
    full = _full_step(kind, engine, gpus, det)
    assert not sel_calls                                   # everything trainable: the entry points of before
    got = _step(kind, engine, gpus, det, fu.PATTERNS[pattern])
    trainable, (lat, cams, rays) = fu.PATTERNS[pattern]
    wanted = {k: trainable(*k.split("/")) for k in got if "/" in k}
    # a frozen parameter takes the selective entry point; with every parameter trainable (only the encoder frozen) the
    # node calls what it called before, and so does the sharded node of a wholly frozen network
    sel = ["pnr_render_backward_sel" if gpus is None else "pnr_mgpu_render_backward_sel"]
    partly = not all(wanted.values()) and (gpus is None or any(wanted.values()))
    assert sel_calls == (sel if partly else [])
    wanted.update(latent=lat, poses=cams, focal=cams, c=cams, rays=rays)
    for k, want in wanted.items():
        if not want:
            assert got[k] is None, k
            continue
        assert got[k] is not None, k
        if det:
            assert torch.equal(got[k], full[k]), (k, rel(got[k], full[k]))
        else:
            assert rel(got[k], full[k]) <= 1e-5, (k, rel(got[k], full[k]))
    if kind != "tiny":
        assert any(got[k].abs().max() > 0 for k, want in wanted.items() if want)


def test_field_node_with_frozen_layers():
    """net(xyz) in grad mode with only blocks 3-4 and lin_out trainable: pnr_field_backward_sel, bit-equal (deterministic
    mode) to the all-trainable node for those tensors and xyz; the rest keep .grad None."""
    import gpu_util
    case = gu.load_case("sb2_d")
    cfg = case["cfg"]
    g = torch.Generator().manual_seed(2)
    r = case["rays"][:, :10]
    xyz0 = (r[..., :3] + (0.8 + torch.rand(cfg["SB"], 10, 1, generator=g)) * r[..., 3:6]).contiguous()
    d_out = (torch.randn(cfg["SB"], 10, 4, generator=g) * 1e-2).cuda()
    trainable = fu.PATTERNS["blocks_3_4_and_lin_out"][0]
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        res = []
        for frozen in (False, True):
            net = gpu_util.build_net(case, device="cuda:0", engine="auto").train()
            for k, p in net.mlp_coarse.named_parameters():
                p.requires_grad_(not frozen or trainable("c", k))
            xyz = xyz0.cuda().requires_grad_(True)
            net(xyz, coarse=True, viewdirs=r[..., 3:6].cuda()).backward(d_out)
            res.append(({k: p.grad for k, p in net.mlp_coarse.named_parameters()}, xyz.grad))
    finally:
        torch.use_deterministic_algorithms(prev)
    (full, fx), (sel, sx) = res
    assert torch.equal(fx, sx)
    for k, v in sel.items():
        if trainable("c", k):
            assert torch.equal(v, full[k]), k
        else:
            assert v is None, k
