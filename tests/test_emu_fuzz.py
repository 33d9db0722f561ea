"""Randomised differential test of the CUDA sources (SIMT path, run on the host emulator of tests/cuda_emu) against the
oracle: random object / view / image / latent sizes, focal and principal-point formats, sample counts and background
modes -- forward through pnr_render, backward through pnr_render_backward.  Deterministic (seeded)."""
import os
import random

import pytest
import torch

import emu_util as eu
import golden_util as gu
from test_emu_kernels import _emulated_training_step, fine_checked, rel

bw = gu.load_by_path("pnr_backward", os.path.join(gu.ROOT, "oracle", "pnr_backward.py"))
synth, oracle = gu.synth, gu.oracle


def random_case(seed):
    rnd = random.Random(seed)
    SB, NS = rnd.randint(1, 3), rnd.randint(1, 4)
    W, H = rnd.randint(8, 24), rnd.randint(8, 24)
    Hl, Wl = rnd.randint(4, 10), rnd.randint(4, 10)
    Kc = rnd.randint(2, 10)
    Kf = 0 if rnd.random() < 0.2 else rnd.randint(1, 8)
    Kfd = rnd.randint(0, Kf)
    B = rnd.randint(1, 7)
    d_hidden = rnd.choice([16, 32, 48])
    z_near, z_far = 0.8, 1.8
    r = 1.3
    f0 = 0.9 * W
    fmt = rnd.choice(["scalar", "per_object", "fxfy"])
    if fmt == "scalar":
        focal = torch.tensor(f0)
    elif fmt == "per_object":
        focal = torch.tensor([f0 * (1.0 + 0.1 * o) for o in range(SB)])
    else:
        focal = torch.tensor([[f0 * (1.0 + 0.1 * o), f0 * 1.07] for o in range(SB)])
    cfmt = rnd.choice(["none", "shared", "per_object"])
    c = None if cfmt == "none" else torch.tensor(
        [[W * 0.5 + 0.7 * o, H * 0.5 - 0.4] for o in range(SB if cfmt == "per_object" else 1)])
    src = torch.stack([torch.stack([synth.pose_spherical(rnd.uniform(0, 360), rnd.uniform(-60, -5), r)
                                    for _ in range(NS)]) for _ in range(SB)])
    tgt = torch.stack([synth.pose_spherical(rnd.uniform(0, 360), rnd.uniform(-40, -5), r) for _ in range(SB)])
    all_rays = synth.gen_rays(tgt, W, H, float(f0), z_near, z_far)
    g = torch.Generator().manual_seed(seed)
    pix = torch.randint(0, W * H, (SB, B), generator=g)
    rays = torch.stack([all_rays[o].reshape(-1, 8)[pix[o]] for o in range(SB)]).contiguous()
    cfg = dict(SB=SB, NS=NS, W=W, H=H, Hl=Hl, Wl=Wl, n_coarse=Kc, n_fine=Kf, n_fine_depth=Kfd, B=B,
               d_hidden=d_hidden, white_bkgd=rnd.random() < 0.5, eval_batch_size=50000)
    return dict(name=f"fuzz{seed}", cfg=cfg, seed=seed, src_poses=src,
                latent=(synth.make_latent(seed, SB * NS, Hl, Wl) * 0.05).contiguous(), focal=focal, c=c, rays=rays,
                wc=synth.make_mlp_weights(seed + 2, d_hidden),
                wf=synth.make_mlp_weights(seed + 3, d_hidden) if (Kf > 0 and rnd.random() < 0.7) else None,
                noise=synth.draw_noise(seed + 4, SB * B, Kc, Kf, Kfd))


@pytest.mark.parametrize("seed", list(range(100, 124)))
def test_random_configuration(seed):
    case = random_case(seed)
    cfg = case["cfg"]
    gt = torch.rand(cfg["SB"], cfg["B"], 3, generator=torch.Generator().manual_seed(seed + 9))
    loss, g_c, g_f, d_lat, t = _emulated_training_step(case, gt)
    ref = gu.oracle_render(case)
    assert (t["z_coarse"] - ref["coarse"]["z"]).abs().max() < 1e-6
    assert (t["rgb_coarse"] - ref["coarse"]["rgb"]).abs().max() < 1e-4
    assert (t["weights_coarse"] - ref["coarse"]["weights"]).abs().max() < 1e-4
    if cfg["n_fine"] > 0:
        fine_checked(case, t)
        if ((t["z_fine"] - ref["fine"]["z"]).abs() > 2e-4).any():
            # the forward was checked above on the emulator's own samples; the oracle backward below replays the
            # oracle's samples, so its gradients are comparable only where both took the same bins
            pytest.skip("an importance sample took a bin next to the oracle's: gradients are not comparable")
    m_loss, o_c, o_f, o_lat = bw.train_loss_backward(case["rays"], gt, case["noise"], gu.oracle_state(case),
                                                     case["latent"], case["wc"], case["wf"], cfg["NS"],
                                                     cfg["n_coarse"], cfg["n_fine"], cfg["n_fine_depth"],
                                                     white_bkgd=cfg["white_bkgd"])
    assert abs(loss - m_loss.item()) < 1e-5

    def close(a, b, what):
        if float(b.abs().max()) == 0.0:
            assert float(a.abs().max()) < 1e-12, what
        else:
            assert rel(a, b) < 5e-4, what

    close(d_lat, o_lat, "latent")
    for k in o_c:
        close(g_c[k], o_c[k], ("coarse", k))
    if o_f is not None:
        for k in o_f:
            close(g_f[k], o_f[k], ("fine", k))
