"""TEST INFRASTRUCTURE: runs the UNMODIFIED reference in its own interpreter (its packages are called `model`, `render`,
`util` like this repo's, so the two cannot share one) and dumps what a test needs into a .pt file.

  python tests/ref_probe.py checkpoint <dir>      a checkpoint written by the reference's own save_weights (row f-4)
  python tests/ref_probe.py load <dir>            the reference strict-loads <dir>/ours/pixel_nerf_latest (written by us)
"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_harness as rh  # noqa: E402


def scene(seed, SB, NS, H, W):
    g = torch.Generator().manual_seed(seed)
    images = torch.rand(SB, NS, 3, H, W, generator=g) * 2 - 1
    poses = torch.eye(4).repeat(SB, NS, 1, 1)
    poses[..., :3, :3] = torch.linalg.qr(torch.randn(SB, NS, 3, 3, generator=g))[0]
    poses[..., :3, 3] = torch.randn(SB, NS, 3, generator=g)
    focal = torch.rand(SB, 2, generator=g) * 50 + 40
    c = torch.rand(SB, 2, generator=g) * 4 + torch.tensor([W / 2.0, H / 2.0])
    return images, poses, focal, c


class _Args:
    def __init__(self, d, name="probe", resume=True):
        self.checkpoints_path, self.name, self.resume = d, name, resume


def cmd_checkpoint(d):
    """The reference's own `save_weights` (models.py:300-316) on a perturbed random-init net + the field values its own
    forward gives for that checkpoint on a small scene."""
    model, render, _ = rh.import_reference()
    torch.manual_seed(11)
    net = model.make_model(rh.model_conf(512, True)).eval()
    with torch.no_grad():
        for mlp in (net.mlp_coarse, net.mlp_fine):
            for blk in mlp.blocks:
                blk.fc_1.weight.normal_(0, 0.03)
            mlp.lin_out.bias[3] = 1.0
    os.makedirs(os.path.join(d, "probe"), exist_ok=True)
    net.save_weights(_Args(d))
    net.save_weights(_Args(d))            # second save rolls the backup file (models.py:307-314)
    images, poses, focal, c = scene(5, 1, 2, 32, 32)
    with torch.no_grad():
        net.encode(images, poses, focal, c=c)
        xyz = torch.randn(1, 64, 3) * 0.4
        dirs = torch.nn.functional.normalize(torch.randn(1, 64, 3), dim=-1)
        out_c = net(xyz, coarse=True, viewdirs=dirs)
        out_f = net(xyz, coarse=False, viewdirs=dirs)
    torch.save(dict(images=images, poses=poses, focal=focal, c=c, xyz=xyz, dirs=dirs, out_coarse=out_c, out_fine=out_f,
                    keys=list(net.state_dict().keys())), os.path.join(d, "probe_io.pt"))


def cmd_load(d):
    """Strict-load a checkpoint (written by THIS repo's save_weights) with the reference's own load_weights."""
    model, _, _ = rh.import_reference()
    net = model.make_model(rh.model_conf(512, True))
    before = net.mlp_coarse.lin_in.weight.clone()
    net.load_weights(_Args(d, name="ours"), strict=True)
    assert not torch.equal(before, net.mlp_coarse.lin_in.weight), "checkpoint was not loaded"
    io = torch.load(os.path.join(d, "probe_io.pt"))
    with torch.no_grad():
        net.eval()
        net.encode(io["images"], io["poses"], io["focal"], c=io["c"])
        out = net(io["xyz"], coarse=True, viewdirs=io["dirs"])
    print("MAXDIFF", (out - io["out_coarse"]).abs().max().item())


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("cmd", choices=["checkpoint", "load"])
    ap.add_argument("out")
    a = ap.parse_args()
    {"checkpoint": cmd_checkpoint, "load": cmd_load}[a.cmd](a.out)
