"""Fused forward + `pnr_field_backward` for PixelNeRFNet.forward in grad mode on CUDA (SURVEY 8f-1).

Used whenever `net(xyz, ...)` itself is called with gradients required (a whole training step through
`NeRFRenderer` uses the render-level node of render/fused_train.py instead; `PNR_FUSED_BACKWARD=1` forces this
field-level node there too, `=0` the composed-torch path).  Validated on H100 (tests/test_gpu_backward.py).

The autograd node takes the sample positions, the latent and the MLP parameters as inputs, so autograd carries
`d_xyz` back into the renderer (sample depths), `d_latent` into the encoder trunk and the weight gradients into the
optimiser, exactly where the reference's graph has them (train/train.py:199-215).
"""
import torch

import pnr_native as pn


class _FusedField(torch.autograd.Function):
    @staticmethod
    def forward(ctx, net, coarse, xyz, viewdirs, latent, *params):
        ctx.net, ctx.coarse = net, coarse
        ctx.save_for_backward(xyz, viewdirs)
        with torch.no_grad():
            return net._field_fused(xyz, coarse, viewdirs)

    @staticmethod
    def backward(ctx, d_out):
        net, coarse = ctx.net, ctx.coarse
        xyz, viewdirs = ctx.saved_tensors
        SB, B, _ = xyz.shape
        use_fine = (not coarse) and net.mlp_fine is not None
        mlp = net.mlp_fine if use_fine else net.mlp_coarse
        scene, mc, mf, keep = net._scene_struct(want_fine=use_fine)
        m = mf if use_fine else mc
        dev = xyz.device
        names = [k for k, _ in mlp.named_parameters()]
        grads = {k: torch.zeros_like(p, dtype=torch.float32, memory_format=torch.contiguous_format)
                 for k, p in mlp.named_parameters()}
        gstruct = pn.make_mlp_struct(grads, mlp.d_in, mlp.d_latent, mlp.d_hidden, mlp.d_out, mlp.n_blocks,
                                     mlp.combine_layer)
        V, C, Hl, Wl = net.encoder.latent.shape
        want_latent = ctx.needs_input_grad[4]
        d_latent = torch.zeros(V, Hl, Wl, C, dtype=torch.float32, device=dev) if want_latent else None
        d_xyz = torch.empty(SB, B, 3, dtype=torch.float32, device=dev) if ctx.needs_input_grad[2] else None
        xyz_c = xyz.detach().contiguous().float()
        dirs_c = viewdirs.detach().reshape(SB, B, 3).contiguous().float()
        d_out_c = d_out.contiguous().float()
        L = pn.lib()
        nbytes = L.pnr_field_backward_workspace_bytes(scene, m, B)
        ws = pn.workspace(dev, nbytes)
        with torch.cuda.device(dev):
            pn.check(L.pnr_field_backward(scene, m, pn.dptr(xyz_c, "xyz"), pn.dptr(dirs_c, "viewdirs"),
                                          pn.dptr(d_out_c, "d_out"), gstruct, pn.dptr(d_latent), pn.dptr(d_xyz), B,
                                          ws.data_ptr(), ws.numel(), pn.stream_ptr(dev)))
        g_latent = d_latent.permute(0, 3, 1, 2) if want_latent else None
        return (None, None, d_xyz, None, g_latent) + tuple(grads[k] for k in names)


def fused_field(net, xyz, coarse, viewdirs):
    use_fine = (not coarse) and net.mlp_fine is not None
    mlp = net.mlp_fine if use_fine else net.mlp_coarse
    latent = net.encoder.latent.detach() if net.stop_encoder_grad else net.encoder.latent
    params = [p for _, p in mlp.named_parameters()]
    return _FusedField.apply(net, coarse, xyz, viewdirs, latent, *params)
