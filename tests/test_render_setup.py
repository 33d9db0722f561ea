"""Setup of the fused render call on the CPU (render/fused_call.py): the draws and their order, the rows a shard takes
of injected draws, and the wiring of the output tensors into PnrRenderOut and of the draws into PnrNoise."""
import ctypes as C
import os
import sys
from types import SimpleNamespace

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pixel-nerf_b200", "src"))

import pnr_native as pn  # noqa: E402
from render import fused_call as fc  # noqa: E402
from render.sharding import shard_bounds  # noqa: E402

# (n_coarse, n_fine, n_fine_depth, using_fine): importance and depth samples, no depth samples, depth samples only,
# fine pass switched off, no fine samples
RENDERERS = [(5, 4, 2, True), (5, 4, 0, True), (5, 3, 3, True), (5, 4, 2, False), (5, 0, 0, True)]


def _renderer(Kc, Kf, Kfd, using_fine):
    return SimpleNamespace(n_coarse=Kc, n_fine=Kf, n_fine_depth=Kfd, using_fine=using_fine)


@pytest.fixture
def cpu_dptr(monkeypatch):
    """pn.dptr accepting CPU tensors, so the structs can be filled without a GPU."""
    monkeypatch.setattr(pn, "dptr", lambda t, name="tensor": None if t is None else C.c_void_p(t.data_ptr()))


@pytest.mark.parametrize("cfg", RENDERERS)
def test_draws_follow_the_reference_order(cfg, cpu_dptr):
    Kc, Kf, Kfd, using_fine = cfg
    counts = fc.sample_counts(_renderer(*cfg))
    fine = using_fine and Kf > 0
    assert counts == ((Kc, Kf, Kfd, True) if fine else (Kc, 0, 0, False))
    R = 6
    torch.manual_seed(3)
    draws = fc.draw_noise(R, counts, "cpu")
    after = torch.rand(1)
    torch.manual_seed(3)
    ref = {"u_coarse": torch.rand(R, Kc)}
    if fine and Kf - Kfd > 0:
        ref["u_fine"] = torch.rand(R, Kf - Kfd)
        ref["u_fine_jit"] = torch.rand(R, Kf - Kfd)
    if fine and Kfd > 0:
        ref["n_depth"] = torch.randn(R, Kfd)
    assert torch.equal(torch.rand(1), after)            # the same number of draws
    assert draws.keys() == ref.keys()
    for k in ref:
        assert torch.equal(draws[k], ref[k]), k

    lin = torch.linspace(0, 1 - 1.0 / Kc, Kc)
    noise = fc.bind_noise(lin, draws)
    assert noise.lin_steps == lin.data_ptr()
    for k in ("u_coarse", "u_fine", "u_fine_jit", "n_depth"):
        assert getattr(noise, k) == (draws[k].data_ptr() if k in draws else None), k


@pytest.mark.parametrize("cfg", RENDERERS)
def test_injected_draws_are_replayed_as_fp32(cfg):
    counts = fc.sample_counts(_renderer(*cfg))
    Kc, Kf, Kfd, _ = counts
    R = 6
    g = torch.Generator().manual_seed(1)
    full = {"u_coarse": torch.rand(Kc, R, generator=g, dtype=torch.float64).t(),
            "u_fine": torch.rand(R, 4, generator=g), "u_fine_jit": torch.rand(R, 4, generator=g),
            "n_depth": torch.randn(R, 2, generator=g)}
    draws = fc.draw_noise(R, counts, "cpu", noise_in=full)
    used = ["u_coarse"] + (["u_fine", "u_fine_jit"] if Kf - Kfd > 0 else []) + (["n_depth"] if Kfd > 0 else [])
    assert sorted(draws) == sorted(used)
    for k in used:
        assert draws[k].dtype == torch.float32 and draws[k].is_contiguous()
        assert torch.equal(draws[k], full[k].float()), k


@pytest.mark.parametrize("SB,B,n", [(1, 7, 3), (2, 7, 3), (3, 2, 4), (2, 9, 2)])
def test_shard_rows_of_injected_draws(SB, B, n):
    """Each shard [a, b) takes rows v.reshape(SB, B, -1)[:, a:b] of the full-ray draws: ragged and empty shards."""
    counts = (4, 3, 1, True)
    g = torch.Generator().manual_seed(2)
    full = {"u_coarse": torch.rand(SB * B, 4, generator=g), "u_fine": torch.rand(SB * B, 2, generator=g),
            "u_fine_jit": torch.rand(SB * B, 2, generator=g), "n_depth": torch.randn(SB * B, 1, generator=g)}
    bounds = shard_bounds(B, n)
    assert any(b == a for a, b in bounds) == (n > B)
    for a, b in bounds:
        draws = fc.draw_noise(SB * (b - a), counts, "cpu", noise_in=full, rows=(SB, B, a, b))
        assert sorted(draws) == sorted(full)
        for k, v in full.items():
            ref = v.reshape(SB, B, -1)[:, a:b]
            assert draws[k].shape == (SB * (b - a), v.shape[1]), (k, a, b)
            assert torch.equal(draws[k].reshape(ref.shape), ref), (k, a, b)


FIELDS = {"rgb_coarse": ("coarse", "rgb"), "depth_coarse": ("coarse", "depth"),
          "weights_coarse": ("coarse", "weights"), "z_coarse": ("coarse", "z"),
          "rgb_fine": ("fine", "rgb"), "depth_fine": ("fine", "depth"),
          "weights_fine": ("fine", "weights"), "z_fine": ("fine", "z")}


@pytest.mark.parametrize("want_weights", [False, True])
@pytest.mark.parametrize("want_z", [False, True])
@pytest.mark.parametrize("fine", [False, True])
@pytest.mark.parametrize("SB", [1, 3])
def test_outputs_are_what_the_struct_points_at(want_weights, want_z, fine, SB, cpu_dptr):
    B, Kc, Kf = 5, 4, 6
    counts = (Kc, Kf, 2, True) if fine else (Kc, 0, 0, False)
    out, res = fc.render_outputs(SB, B, counts, "cpu", want_weights, want_z)
    shapes = {"rgb": (3,), "depth": (), "weights": None, "z": None}
    expect = {"rgb", "depth"} | ({"weights"} if want_weights else set()) | ({"z"} if want_z else set())
    assert set(res) == ({"coarse", "fine"} if fine else {"coarse"})
    for p, K in (("coarse", Kc), ("fine", Kc + Kf)):
        if p not in res:
            continue
        assert set(res[p]) == expect
        for q, t in res[p].items():
            assert t.dtype == torch.float32 and t.is_contiguous()
            assert t.shape == (SB, B) + (shapes[q] if shapes[q] is not None else (K,)), (p, q)
    ptrs = []
    for field, (p, q) in FIELDS.items():
        t = res[p][q] if p in res and q in res[p] else None
        assert getattr(out, field) == (None if t is None else t.data_ptr()), field
        ptrs += [] if t is None else [t.data_ptr()]
    assert len(set(ptrs)) == len(ptrs)                  # no two outputs share storage
