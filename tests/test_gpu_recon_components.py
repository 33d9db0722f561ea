"""Connected components on the H100: pnr_mesh_components bit for bit against the oracle (oracle/pnr_recon_components.py)
on random soups of 12 M triangles whose components range from single vertices to one spanning half the vertices, the
same bits from two calls (the hooking runs concurrently only here), the analytic sphere scene through the GPU marching
cubes, `util.recon.keep_components` on what `marching_cubes` and `fuse_views` return for the C2 scene, and the
refusals."""
import numpy as np
import pytest
import torch

from components_util import BIG, SMALL, bits_equal, comp, random_soup, sphere_field
from test_gpu_recon import C1_, C2_, c2_net
from test_gpu_recon import _Spy as _VolSpy

pytestmark = pytest.mark.gpu


def big_soup(seed, n_verts=6_000_000, n_tris=12_000_000):
    g = np.random.default_rng(seed)
    sizes = np.concatenate([[n_verts // 2], g.integers(1, 2000, size=n_verts // 1000), np.ones(n_verts, np.int64)])
    return random_soup(seed, n_verts, n_tris, sizes=sizes), n_verts


def test_labels_and_counts_bit_equal_on_large_soups():
    import pnr_native as pn
    for seed in (1, 2):
        tris, n = big_soup(seed)
        t = torch.from_numpy(tris).cuda()
        label, tri_count, count = pn.mesh_components(t, n)
        want_label = comp.labels(tris, n)
        want_count = comp.tri_counts(tris, want_label)
        label, tri_count = label.cpu().numpy(), tri_count.cpu().numpy()
        sizes = np.bincount(want_label, minlength=n)
        print(f"seed {seed}: {count} components with triangles, largest {sizes.max()} of {n} vertices, "
              f"{np.count_nonzero(sizes == 1)} single vertices")
        assert sizes.max() >= n // 3 and (sizes == 1).sum() > 1000 and count > 1000
        assert bits_equal(label, want_label)
        assert bits_equal(tri_count, want_count)
        assert count == np.count_nonzero(want_count)
        label2, tri_count2, count2 = pn.mesh_components(t, n)           # the same bits again
        assert bits_equal(label2.cpu().numpy(), label) and bits_equal(tri_count2.cpu().numpy(), tri_count)
        assert count2 == count
        # the compaction of the 3 largest, against the oracle's
        keep_root = np.zeros(n, dtype=np.uint8)
        keep_root[comp.kept_roots(want_count, 3)] = 1
        vert_ids, tris_out = pn.mesh_compact(t, n, torch.from_numpy(label).cuda(), torch.from_numpy(keep_root).cuda())
        want_v, want_t = comp.keep_components(np.arange(n)[:, None], tris, largest=3)
        assert bits_equal(vert_ids.cpu().numpy(), want_v[:, 0]) and bits_equal(tris_out.cpu().numpy(), want_t)


def test_sphere_scene_through_the_gpu_marching_cubes():
    import pnr_native as pn
    from util import recon as urecon
    v, t = (a.cpu().numpy() for a in pn.marching_cubes(torch.from_numpy(sphere_field([BIG] + SMALL)).cuda(), 0.0))
    big = [a.cpu().numpy() for a in pn.marching_cubes(torch.from_numpy(sphere_field([BIG])).cuda(), 0.0)]
    kv, kt = urecon.keep_components(v, t, largest=1)
    assert bits_equal(kv, big[0]) and bits_equal(kt, big[1])
    sizes = {s[1]: len(pn.marching_cubes(torch.from_numpy(sphere_field([s])).cuda(), 0.0)[1]) for s in SMALL}
    for k in sorted(sizes.values()):
        kv, kt = urecon.keep_components(v, t, largest=None, min_triangles=k)
        want = pn.marching_cubes(torch.from_numpy(sphere_field([BIG] + [s for s in SMALL if sizes[s[1]] >= k])).cuda(),
                                 0.0)
        assert bits_equal(kv, want[0].cpu().numpy()) and bits_equal(kt, want[1].cpu().numpy()), k
    everything = urecon.keep_components(v, t, largest=None)
    assert bits_equal(everything[0], v) and bits_equal(everything[1], t)


def assert_matches_oracle(mesh, **kw):
    from util import recon as urecon
    got = urecon.keep_components(*mesh, **kw)
    want = comp.keep_components(*mesh, **kw)
    assert len(got) == len(want) == len(mesh)
    for a, b in zip(got, want):
        assert bits_equal(a, b)
    return got


def test_keep_components_of_marching_cubes_on_c2_scene(monkeypatch):
    from util import recon as urecon
    net, _, _ = c2_net("tc")
    spy = _VolSpy(monkeypatch)
    urecon.marching_cubes(net, C1_, C2_, [12, 12, 12], isosurface=1e9)
    iso = float(np.quantile(spy.vols[-1], 0.7))          # a level the field crosses
    monkeypatch.undo()
    mesh = urecon.marching_cubes(net, C1_, C2_, [40, 36, 44], isosurface=iso, return_colors=True)
    label = comp.labels(mesh[1], len(mesh[0]))
    print(f"{len(mesh[1])} triangles in {np.count_nonzero(comp.tri_counts(mesh[1], label))} components")
    assert len(mesh[1]) > 1000
    kept = assert_matches_oracle(mesh, largest=1)
    assert 0 < len(kept[1]) <= len(mesh[1]) and kept[2].dtype == np.float64 and kept[3].dtype == np.float32
    assert_matches_oracle(mesh, largest=None, min_triangles=20)
    for a, b in zip(urecon.keep_components(*mesh, largest=None), mesh):  # every vertex is used: the mesh comes back
        assert bits_equal(a, b)


def test_keep_components_of_fuse_views_on_c2_scene(monkeypatch):
    from test_gpu_recon_fuse import c2_scene
    from test_gpu_recon_paint import _Spy as _PaintSpy
    from test_gpu_recon_paint import call
    net, renderer, poses = c2_scene()
    spy = _PaintSpy(monkeypatch)
    call(net, renderer, poses)
    m = float(np.clip(np.median(spy.fused[-1][1]), 0.05, 1.0))           # an opacity level the scene crosses
    mesh = call(net, renderer, poses, min_opacity=m, return_colors=True, colors="views")
    label = comp.labels(mesh[1], len(mesh[0]))
    print(f"{len(mesh[1])} triangles in {np.count_nonzero(comp.tri_counts(mesh[1], label))} components")
    assert len(mesh[1]) > 100
    assert_matches_oracle(mesh, largest=1)
    assert_matches_oracle(mesh, largest=2, min_triangles=8)


def test_refusals():
    from util import recon as urecon
    v = np.zeros((4, 3))
    t = np.array([[0, 1, 2], [1, 2, 3]])
    for kw in (dict(largest=0), dict(largest=-1), dict(largest=1.5), dict(largest=True), dict(min_triangles=0),
               dict(min_triangles=None)):
        with pytest.raises(ValueError, match="largest|min_triangles"):
            urecon.keep_components(v, t, **kw)
    for args in ((np.zeros((4, 2)), t), (np.zeros(12), t), (v, t[:, :2]), (v, t.astype(np.float64)),
                 (v, t, np.zeros((3, 3))), (v, t, np.zeros(())), (v, np.array([[0, 1, 4]])),
                 (v, np.array([[0, -1, 2]])), (v, np.array([[0, 1, 2], [2 ** 40, 0, 1]]))):
        with pytest.raises(ValueError):
            urecon.keep_components(*args)
    with pytest.raises(RuntimeError, match="CUDA"):
        urecon.keep_components(v, t, device="cpu")
