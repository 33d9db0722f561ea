"""Training steps of a partly frozen network through the public classes (NeRFRenderer.bind_parallel in train mode), for
tests/test_gpu_frozen.py and scripts/bench_frozen.py: the freeze patterns, the C2 train-shape scene (SB = 4 objects,
B = 128 rays, train/train.py's defaults) and the golden-case scenes."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "tests"), os.path.join(ROOT, "pixel-nerf_b200", "src")):
    if p not in sys.path:
        sys.path.insert(0, p)

import golden_util as gu  # noqa: E402
import gpu_util  # noqa: E402

# name -> (is (mlp "c"/"f", parameter name) trainable, (latent, cameras, rays) trainable)
PATTERNS = {
    "network_frozen_rays_poses": (lambda m, k: False, (False, True, True)),     # pose refinement
    "encoder_frozen": (lambda m, k: True, (False, False, False)),               # train.py --freeze_enc
    "coarse_frozen": (lambda m, k: m == "f", (True, False, False)),
    "fine_frozen": (lambda m, k: m == "c", (True, False, False)),
    "blocks_3_4_and_lin_out": (lambda m, k: k.startswith(("blocks.3.", "blocks.4.", "lin_out.")), (False, False, False)),
    "lin_in_only": (lambda m, k: k.startswith("lin_in."), (False, False, False)),
    "biases_only": (lambda m, k: k.endswith(".bias"), (False, False, False)),
}
FULL = (lambda m, k: True, (True, True, True))


class Scene:
    """A model, renderer, latent, source cameras, rays and an rgb target on `dev`.  kind: "c2" (the C2 model,
    d_hidden 512, at the train shape) or a golden case name."""

    def __init__(self, kind, dev):
        from model import make_model
        from render import NeRFRenderer
        g = torch.Generator().manual_seed(7)
        if kind == "c2":
            c2 = gu.synth.CONFIGS["c2"]
            SB, NS, B = 4, c2["NS"], 128
            net = make_model(gpu_util.model_conf(512))
            net.mlp_coarse.load_state_dict(gu.synth.make_mlp_weights(31, 512))
            net.mlp_fine.load_state_dict(gu.synth.make_mlp_weights(32, 512))
            self.W, self.H = c2["W"], c2["H"]
            r = (c2["z_near"] + c2["z_far"]) * 0.5
            self.src = torch.stack([torch.stack([gu.synth.pose_spherical(40.0 * v + 25.0 * o, -30.0, r)
                                                 for v in range(NS)]) for o in range(SB)])
            self.latent = gu.synth.make_latent(5, SB * NS, 32, 32)
            self.focal = torch.tensor([c2["focal"]])
            tgt = torch.stack([gu.synth.pose_spherical(100.0 + 70.0 * o, -10.0 - 5 * o, r) for o in range(SB)])
            all_rays = gu.synth.gen_rays(tgt, self.W, self.H, torch.tensor(c2["focal"]), c2["z_near"],
                                         c2["z_far"]).reshape(SB, -1, 8)
            pix = torch.randint(0, self.W * self.H, (SB, B), generator=g)
            self.rays = torch.gather(all_rays, 1, pix[..., None].expand(-1, -1, 8)).contiguous()
            renderer = NeRFRenderer(n_coarse=c2["n_coarse"], n_fine=c2["n_fine"], n_fine_depth=c2["n_fine_depth"],
                                    depth_std=0.01, white_bkgd=c2["white_bkgd"])
        else:
            case = gu.load_case(kind)
            cfg = case["cfg"]
            net = gpu_util.build_net(case, device="cpu")
            self.W, self.H = cfg["W"], cfg["H"]
            self.src, self.latent, self.focal = case["src_poses"], case["latent"], case["focal"]
            self.rays = case["rays"].contiguous()
            renderer = gpu_util.build_renderer(case)
            SB, B = self.rays.shape[:2]
        self.c = torch.tensor([[self.W * 0.5, self.H * 0.5]])
        self.target = torch.rand(SB, B, 3, generator=g)
        self.net, self.renderer = net.to(dev).train(), renderer.to(dev).train()
        for name in ("src", "latent", "focal", "c", "rays", "target"):
            setattr(self, name, getattr(self, name).to(dev).float())

    def mlps(self):
        return [(t, m) for t, m in (("c", self.net.mlp_coarse), ("f", self.net.mlp_fine)) if m is not None]

    def step(self, pattern, gpus=None, engine="tc", events=None):
        """One training step (render with want_weights, MSE coarse + MSE fine, backward) with `pattern`'s tensors
        trainable -> dict: "c/<name>", "f/<name>" parameter gradients, latent, poses, focal, c, rays (.grad or None).
        events: optional (start, end) CUDA events recorded around loss.backward()."""
        trainable, (lat, cams, rays_w) = pattern
        net = self.net
        net.engine = engine
        for tag, mlp in self.mlps():
            for k, p in mlp.named_parameters():
                p.requires_grad_(trainable(tag, k))
                p.grad = None
        latent = self.latent.clone().requires_grad_(lat)
        src, focal, c = (t.clone().requires_grad_(cams) for t in (self.src, self.focal, self.c))
        rays = self.rays.clone().requires_grad_(rays_w)
        net.set_scene(latent, src, focal, c, self.W, self.H)
        torch.manual_seed(12)
        out = self.renderer.bind_parallel(net, gpus).train()(rays, want_weights=True)
        loss = ((out["fine"]["rgb"] - self.target) ** 2).mean() + ((out["coarse"]["rgb"] - self.target) ** 2).mean()
        if events:
            events[0].record()
        loss.backward()
        if events:
            events[1].record()
        res = {f"{tag}/{k}": p.grad for tag, mlp in self.mlps() for k, p in mlp.named_parameters()}
        res.update(latent=latent.grad, poses=src.grad, focal=focal.grad, c=c.grad, rays=rays.grad)
        return res
