"""Cost of deterministic mode (torch.use_deterministic_algorithms(True)) on the training step.

At the C2 train shape (SB = 4 objects x NS = 2 views of 128 x 128, B = 128 rays each, tensor engine, encoder
trained): device time of loss.backward() for train.py's loss (MSE coarse + fine, want_weights), device time of the
encoder's backward alone (autograd from the latent), and the peak memory of each, with the flag off and on, alternating
in one process.  Prints one JSON line with the card's name and power limit.

    CUBLAS_WORKSPACE_CONFIG=:4096:8 python scripts/bench_deterministic.py --iters 20
"""
import argparse
import json
import os
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "tests"), os.path.join(ROOT, "pixel-nerf_b200", "src")]

import torch  # noqa: E402

import golden_util as gu  # noqa: E402
import gpu_util  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name(0)} (power limit unknown: {e})"


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), (torch.cuda.max_memory_allocated() - base) / 2**20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from model import make_model
    from render import NeRFRenderer
    torch.backends.cudnn.benchmark = False
    dev = torch.device("cuda:0")
    c2 = gu.synth.CONFIGS["c2"]
    SB, NS, B = 4, c2["NS"], 128
    torch.manual_seed(0)
    net = make_model(gpu_util.model_conf(512)).to(dev).train()
    net.engine = "tc"
    renderer = NeRFRenderer(n_coarse=c2["n_coarse"], n_fine=c2["n_fine"], n_fine_depth=c2["n_fine_depth"],
                            depth_std=0.01, white_bkgd=c2["white_bkgd"]).to(dev).train()
    r = (c2["z_near"] + c2["z_far"]) * 0.5
    poses = torch.stack([torch.stack([gu.synth.pose_spherical(40.0 * v + 25.0 * o, -30.0, r) for v in range(NS)])
                         for o in range(SB)]).to(dev)
    g = torch.Generator().manual_seed(1)
    images = (torch.rand(SB, NS, 3, c2["H"], c2["W"], generator=g) * 2 - 1).to(dev)
    tgt = torch.stack([gu.synth.pose_spherical(100.0 + 70.0 * o, -10.0, r) for o in range(SB)])
    rays_all = gu.synth.gen_rays(tgt, c2["W"], c2["H"], c2["focal"], c2["z_near"], c2["z_far"]).reshape(SB, -1, 8)
    pix = torch.randint(0, rays_all.shape[1], (SB, B), generator=g)
    rays = torch.stack([rays_all[o][pix[o]] for o in range(SB)]).to(dev)
    gt = torch.rand(SB, B, 3, generator=g).to(dev)
    focal = torch.tensor([c2["focal"]], device=dev)

    def loss_fn():
        net.encode(images, poses, focal)
        out = renderer(net, rays, want_weights=True)
        return ((out["coarse"]["rgb"] - gt) ** 2).mean() + ((out["fine"]["rgb"] - gt) ** 2).mean()

    res = {"off": {"backward_ms": [], "encoder_backward_ms": [], "backward_peak_mib": 0.0,
                   "encoder_backward_peak_mib": 0.0}}
    res["on"] = {k: ([] if isinstance(v, list) else 0.0) for k, v in res["off"].items()}
    for it in range(args.warmup + args.iters):
        for mode in ("off", "on"):
            torch.use_deterministic_algorithms(mode == "on")
            net.zero_grad(set_to_none=True)
            loss = loss_fn()
            ms, mib = timed(loss.backward)
            net.zero_grad(set_to_none=True)
            net.encode(images, poses, focal)
            lat = net.encoder.latent
            up = torch.ones_like(lat) * 1e-3
            ms_e, mib_e = timed(lambda: lat.backward(up))
            if it >= args.warmup:
                d = res[mode]
                d["backward_ms"].append(ms)
                d["encoder_backward_ms"].append(ms_e)
                d["backward_peak_mib"] = max(d["backward_peak_mib"], mib)
                d["encoder_backward_peak_mib"] = max(d["encoder_backward_peak_mib"], mib_e)
    torch.use_deterministic_algorithms(False)
    for d in res.values():
        for k in ("backward_ms", "encoder_backward_ms"):
            v = sorted(d[k])
            d[k] = {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}
    print(json.dumps({"card": card(), "shape": f"SB={SB} NS={NS} B={B} c2 tc encoder trained", **res}))


if __name__ == "__main__":
    main()
