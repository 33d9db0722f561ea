"""State producer and checkpoint compatibility against the UNMODIFIED reference:

  * a19: `SpatialEncoder.forward` / `PixelNeRFNet.encode` -- same state_dict, same images -> the same latent, camera
    state and `index()` values as the reference (src/model/encoder.py:111-164, src/model/models.py:89-144); the
    reference's outputs are stored in tests/golden/encode_state.npz (oracle/make_golden.py);
  * f-4: a checkpoint written by the reference's own `save_weights` strict-loads here and gives the reference's field
    values; a checkpoint written here strict-loads in the reference (src/model/models.py:268-316).  This one runs the
    reference itself (in its own interpreter, tests/ref_probe.py) and needs a checkout.
"""
import os
import subprocess
import sys

import pytest
import torch

import dropin_util as du
import gpu_util

PROBE = os.path.join(du.ROOT, "tests", "ref_probe.py")
needs_ref = pytest.mark.skipif(du.reference_root() is None, reason="no reference checkout (/root/reference or oracle/_ref)")


def probe(*argv):
    env = dict(os.environ)
    env["PIXELNERF_REF"] = du.reference_root()
    r = subprocess.run([sys.executable, PROBE, *argv], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout


class Args:
    def __init__(self, d, name, resume=True):
        self.checkpoints_path, self.name, self.resume = d, name, resume


def test_encoder_and_encode_state_match_the_reference():
    import numpy as np
    from golden_util import GOLD, oracle
    from model import make_model
    z = np.load(os.path.join(GOLD, "encode_state.npz"))
    for name, (use_first_pool, (SB, NS, H, W)) in oracle.ENCODE_CASES.items():
        ref = lambda k: torch.from_numpy(np.asarray(z[name + "/" + k]))
        net = make_model(gpu_util.model_conf(64, use_first_pool)).eval()
        missing = net.load_state_dict(oracle.seeded_state(net.state_dict(), 3), strict=True)
        assert not missing.missing_keys and not missing.unexpected_keys
        images, poses, focal, c, uv = oracle.encode_scene(7, SB, NS, H, W)
        with torch.enable_grad():     # CPU tensors: the composed-torch path (encode() itself has no fused part)
            net.encode(images, poses, focal, c=c)
            idx = net.encoder.index(uv, None, net.image_shape)
        lat = net.encoder.latent.detach()
        assert list(lat.shape) == ref("latent_shape").tolist(), name
        lat_s = lat.reshape(-1)[oracle.encode_sample_index(lat.numel(), 1)]
        assert (lat_s - ref("latent")).abs().max() <= 1e-6 * ref("latent_absmax"), name
        assert torch.equal(net.encoder.latent_scaling, ref("latent_scaling"))
        assert torch.equal(net.poses, ref("poses"))
        assert torch.equal(net.focal, ref("focal")) and torch.equal(net.c, ref("c"))
        assert torch.equal(net.image_shape, ref("image_shape"))
        assert net.num_views_per_obj == int(ref("num_views_per_obj"))
        idx = idx.detach()
        assert list(idx.shape) == ref("index_shape").tolist(), name
        idx_s = idx.reshape(-1)[oracle.encode_sample_index(idx.numel(), 2)]
        assert (idx_s - ref("index")).abs().max() <= 1e-5 * ref("index_absmax"), name


@needs_ref
def test_checkpoints_round_trip_with_the_reference(tmp_path):
    d = str(tmp_path)
    probe("checkpoint", d)
    assert os.path.exists(os.path.join(d, "probe", "pixel_nerf_latest"))
    assert os.path.exists(os.path.join(d, "probe", "pixel_nerf_backup"))
    io = torch.load(os.path.join(d, "probe_io.pt"))
    from model import make_model
    net = make_model(gpu_util.model_conf(512, True)).eval()
    assert list(net.state_dict().keys()) == io["keys"]            # same names, same order
    assert net.load_weights(Args(d, "probe"), strict=True) is net
    with torch.enable_grad():                                      # CPU: composed-torch field
        net.encode(io["images"], io["poses"], io["focal"], c=io["c"])
        oc = net(io["xyz"].requires_grad_(True), coarse=True, viewdirs=io["dirs"]).detach()
        of = net(io["xyz"], coarse=False, viewdirs=io["dirs"]).detach()
    assert (oc - io["out_coarse"]).abs().max() < 1e-5
    assert (of - io["out_fine"]).abs().max() < 1e-5
    # and back: our save_weights -> the reference's load_weights(strict=True) -> its forward gives the same values
    os.makedirs(os.path.join(d, "ours"), exist_ok=True)
    net.save_weights(Args(d, "ours"))
    net.save_weights(Args(d, "ours"))
    assert os.path.exists(os.path.join(d, "ours", "pixel_nerf_backup"))
    out = probe("load", d)
    assert float(out.strip().split("MAXDIFF")[-1]) < 1e-6
    # opt_init semantics (models.py:276-283): no resume + opt_init -> nothing is loaded, returns None
    assert net.load_weights(Args(d, "probe", resume=False), opt_init=True) is None
