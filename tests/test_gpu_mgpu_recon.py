"""Mesh extraction on several GPUs: `util.recon.marching_cubes(..., gpus=...)` (the field passes sharded by
pnr_mgpu_field_eval, csrc/pnr_mgpu_field.cu) against the call without gpus on the C2 scene, bit for bit: vertices,
triangles, normals, colours and every sigma the call evaluated (compared as integers, so NaN equals NaN).  `[0, 0]` and
`[0, 0, 0]` run the whole sharded path -- replicas, the staged stores, empty shards -- on one device; `[0, 1]` needs two
GPUs and is skipped otherwise."""
import numpy as np
import pytest
import torch

from test_gpu_recon import C1_, C2_, c2_net

pytestmark = pytest.mark.gpu


def _two_gpus():
    return torch.cuda.is_available() and torch.cuda.device_count() >= 2


DEVICES = [pytest.param([0, 0], id="one_gpu_two_shards"), pytest.param([0, 0, 0], id="one_gpu_three_shards"),
           pytest.param([0, 1], id="two_gpus", marks=pytest.mark.skipif(not _two_gpus(), reason="needs 2 GPUs"))]

RESO = [40, 36, 44]          # 63360 points


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype, (a.shape, b.shape, a.dtype, b.dtype)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


class _Spy:
    """Records the sigma util.recon hands to marching cubes / the band plan, and the sharded driver calls."""

    def __init__(self, monkeypatch):
        import pnr_native as pn
        from util import recon as urecon
        self.sigma, self.driver, self.fields = [], 0, []
        real_mc, real_plan, real_band, real_eval = pn.marching_cubes, pn.band_plan, pn.band_marching_cubes, \
            pn.mgpu_field_eval

        def mc(vol, iso, **kw):
            self.sigma.append(vol.detach().cpu().numpy().copy())
            return real_mc(vol, iso, **kw)

        def plan(coarse, *a, **kw):
            self.sigma.append(coarse.detach().cpu().numpy().copy())
            return real_plan(coarse, *a, **kw)

        def band_mc(sigma, *a, **kw):
            self.sigma.append(sigma.detach().cpu().numpy().copy())
            return real_band(sigma, *a, **kw)

        def field_eval(*a, **kw):
            self.driver += 1
            return real_eval(*a, **kw)
        monkeypatch.setattr(pn, "marching_cubes", mc)
        monkeypatch.setattr(pn, "band_plan", plan)
        monkeypatch.setattr(pn, "band_marching_cubes", band_mc)
        monkeypatch.setattr(pn, "mgpu_field_eval", field_eval)
        spy = self

        class Field(urecon._ShardedField):
            def __init__(self, *a, **kw):
                super().__init__(*a, **kw)
                spy.fields.append(self)
        monkeypatch.setattr(urecon, "_ShardedField", Field)


_NETS = {}


def net_iso(engine):
    if engine not in _NETS:
        net, _, _ = c2_net(engine)
        g = torch.Generator().manual_seed(0)
        pts = (torch.rand(1, 4096, 3, generator=g) * torch.tensor(C2_) + (1 - torch.rand(1, 4096, 3, generator=g))
               * torch.tensor(C1_)).cuda()
        with torch.no_grad():
            sigma = net(pts, coarse=True, viewdirs=-torch.nn.functional.normalize(pts, dim=-1))[0, :, 3]
        _NETS[engine] = net, float(sigma.median())               # a level the field crosses
    return _NETS[engine]


def extract(net, iso, spy, **kw):
    from util import recon as urecon
    n = len(spy.sigma)
    res = urecon.marching_cubes(net, C1_, C2_, RESO, isosurface=iso, **kw)
    return res, spy.sigma[n:]


CASES = {
    "tc_dense": dict(engine="tc"),
    "tc_dense_colours": dict(engine="tc", return_colors=True),
    "tc_b4_colours": dict(engine="tc", block=4, return_colors=True),
    "tc_b8": dict(engine="tc", block=8),
    "tc_fast_dense_colours": dict(engine="tc_fast", return_colors=True),
    "tc_fast_b4_colours": dict(engine="tc_fast", block=4, return_colors=True),
    "simt_dense_colours": dict(engine="simt", return_colors=True, eval_batch_size=20000),
    "simt_b8": dict(engine="simt", block=8, eval_batch_size=20000),
    "tc_fine_dense_colours": dict(engine="tc", coarse=False, return_colors=True),
    "tc_fine_b4": dict(engine="tc", coarse=False, block=4, return_colors=True),
    "tc_ragged_chunks_b4": dict(engine="tc", eval_batch_size=7777, block=4, return_colors=True),
    "tc_ragged_chunks_dense": dict(engine="tc", eval_batch_size=7777, return_colors=True),
    "tc_one_chunk_empty_shards": dict(engine="tc", eval_batch_size=10 ** 6, return_colors=True),
    "tc_two_chunks": dict(engine="tc", eval_batch_size=50000, return_colors=True),   # [0, 0, 0]: shard 2 empty
}


@pytest.mark.parametrize("devices", DEVICES)
@pytest.mark.parametrize("case", sorted(CASES))
def test_sharded_extraction_is_bit_equal(case, devices, monkeypatch):
    kw = dict(CASES[case])
    net, iso = net_iso(kw.pop("engine"))
    spy = _Spy(monkeypatch)
    ref, ref_sigma = extract(net, iso, spy, **kw)
    assert spy.driver == 0
    got, got_sigma = extract(net, iso, spy, gpus=devices, **kw)
    assert spy.driver == 1 + bool(kw.get("block")) + bool(kw.get("return_colors"))     # every field pass sharded
    assert len(ref[1]) > 1000, len(ref[1])
    assert len(got) == len(ref) == (4 if kw.get("return_colors") else 2)
    for a, b in zip(got, ref):
        same(a, b)
    assert len(got_sigma) == len(ref_sigma)
    for a, b in zip(got_sigma, ref_sigma):
        same(a, b)
    # nothing left behind: the handle is destroyed, the replicas dropped and no shard work outstanding
    field = spy.fields[-1]
    assert field.handle is None and not field.replicas
    for g in set(devices):
        assert torch.cuda.current_stream(torch.device("cuda", g)).query()


@pytest.mark.parametrize("block", [None, 4])
def test_nan_sigma_at_the_origin(block, monkeypatch):
    """An odd grid over a box centred on the origin has a grid point there, whose view direction -p / |p| is NaN:
    the sharded call gives it the same bits as the one-GPU call, whatever the engine makes of it."""
    net, iso = net_iso("tc")
    spy = _Spy(monkeypatch)
    kw = dict(reso=[41, 41, 41], block=block, return_colors=True)
    import util.recon as urecon
    ref = urecon.marching_cubes(net, [-0.5] * 3, [0.5] * 3, isosurface=iso, **kw)
    ref_sigma = spy.sigma[:]
    got = urecon.marching_cubes(net, [-0.5] * 3, [0.5] * 3, isosurface=iso, gpus=[0, 0, 0], **kw)
    got_sigma = spy.sigma[len(ref_sigma):]
    assert len(got_sigma) == len(ref_sigma) == (1 if block is None else 2)
    for a, b in zip(got + tuple(got_sigma), ref + tuple(ref_sigma)):
        same(a, b)


def test_single_device_and_validation(monkeypatch):
    import util.recon as urecon
    net, iso = net_iso("tc")
    spy = _Spy(monkeypatch)
    ref = urecon.marching_cubes(net, C1_, C2_, [20, 18, 22], isosurface=iso)
    got = urecon.marching_cubes(net, C1_, C2_, [20, 18, 22], isosurface=iso, gpus=[0])       # today's path
    assert spy.driver == 0 and not spy.fields
    for a, b in zip(got, ref):
        same(a, b)
    for bad in ([1, 0], [3], []):
        with pytest.raises(ValueError, match="gpus"):
            urecon.marching_cubes(net, C1_, C2_, [10, 10, 10], isosurface=iso, gpus=bad)
    with pytest.raises(RuntimeError, match="CUDA only"):
        urecon.marching_cubes(net, C1_, C2_, [10, 10, 10], device="cpu", gpus=[0, 0])
    net.num_objs = 2
    try:
        with pytest.raises(RuntimeError, match="one object"):
            urecon.marching_cubes(net, C1_, C2_, [10, 10, 10], gpus=[0, 0])
    finally:
        net.num_objs = 1
    assert not spy.fields
