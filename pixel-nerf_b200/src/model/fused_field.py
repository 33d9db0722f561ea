"""Fused forward + `pnr_field_backward` for PixelNeRFNet.forward in grad mode on CUDA (SURVEY 8f-1).

Used whenever `net(xyz, ...)` itself is called with gradients required (a whole training step through
`NeRFRenderer` uses the render-level node of render/fused_train.py instead; `PNR_FUSED_BACKWARD=1` forces this
field-level node there too, `=0` the composed-torch path).  Validated on H100 (tests/test_gpu_backward.py).

The autograd node takes the sample positions, the view directions, the latent, the source cameras (`net.poses`,
`net.focal`, `net.c`) and the MLP parameters as inputs, so autograd carries `d_xyz` / `d_viewdirs` back into the
renderer (sample depths, rays), `d_latent` into the encoder trunk, the camera gradients to the poses / focal / c given
to encode() and the weight gradients into the optimiser, exactly where the reference's graph has them
(train/train.py:199-215, models.py:112-212).  Only the gradients autograd asks for are computed; without view-direction
or camera gradients the backward is `pnr_field_backward`, otherwise `pnr_field_backward_cam`.  With some MLP
parameters frozen (`requires_grad=False`) it is `pnr_field_backward_sel`: the frozen tensors' gradients are neither
allocated nor computed (no weight-gradient GEMM, transposes or bias sum, and no input-gradient chain below the lowest
trainable layer unless an input gradient is wanted) and come back as None; the others are bit-equal to the full call's.
"""
import torch

import pnr_native as pn


class _FusedField(torch.autograd.Function):
    @staticmethod
    def forward(ctx, net, coarse, xyz, viewdirs, latent, poses, focal, c, *params):
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
        wanted = ctx.needs_input_grad[8:]
        grads = {k: torch.zeros_like(p, dtype=torch.float32, memory_format=torch.contiguous_format)
                 for (k, p), w in zip(mlp.named_parameters(), wanted) if w}
        gstruct = pn.make_mlp_struct(grads, mlp.d_in, mlp.d_latent, mlp.d_hidden, mlp.d_out, mlp.n_blocks,
                                     mlp.combine_layer) if grads else None
        V, C, Hl, Wl = net.encoder.latent.shape
        want_latent = ctx.needs_input_grad[4]
        d_latent = torch.zeros(V, Hl, Wl, C, dtype=torch.float32, device=dev) if want_latent else None
        d_xyz = torch.empty(SB, B, 3, dtype=torch.float32, device=dev) if ctx.needs_input_grad[2] else None
        xyz_c = xyz.detach().contiguous().float()
        dirs_c = viewdirs.detach().reshape(SB, B, 3).contiguous().float()
        d_out_c = d_out.contiguous().float()
        d_dirs = torch.empty(SB, B, 3, dtype=torch.float32, device=dev) if ctx.needs_input_grad[3] else None
        cam, d_cam = pn.camera_grad(net, ctx.needs_input_grad[5:8], dev)
        L = pn.lib()
        pn.sync_deterministic()
        nbytes = L.pnr_field_backward_workspace_bytes(scene, m, B)
        ws = pn.workspace(dev, nbytes)
        with torch.cuda.device(dev):
            if not all(wanted):      # part of the MLP is frozen
                pn.check(L.pnr_field_backward_sel(scene, m, pn.dptr(xyz_c, "xyz"), pn.dptr(dirs_c, "viewdirs"),
                                                  pn.dptr(d_out_c, "d_out"), gstruct, pn.dptr(d_latent),
                                                  pn.dptr(d_xyz), pn.dptr(d_dirs), cam, B, ws.data_ptr(), ws.numel(),
                                                  pn.stream_ptr(dev)))
            elif d_dirs is None and cam is None:
                pn.check(L.pnr_field_backward(scene, m, pn.dptr(xyz_c, "xyz"), pn.dptr(dirs_c, "viewdirs"),
                                              pn.dptr(d_out_c, "d_out"), gstruct, pn.dptr(d_latent), pn.dptr(d_xyz),
                                              B, ws.data_ptr(), ws.numel(), pn.stream_ptr(dev)))
            else:
                pn.check(L.pnr_field_backward_cam(scene, m, pn.dptr(xyz_c, "xyz"), pn.dptr(dirs_c, "viewdirs"),
                                                  pn.dptr(d_out_c, "d_out"), gstruct, pn.dptr(d_latent),
                                                  pn.dptr(d_xyz), pn.dptr(d_dirs), cam, B, ws.data_ptr(), ws.numel(),
                                                  pn.stream_ptr(dev)))
        g_latent = d_latent.permute(0, 3, 1, 2) if want_latent else None
        g_dirs = d_dirs.reshape(viewdirs.shape) if d_dirs is not None else None
        return (None, None, d_xyz, g_dirs, g_latent) + d_cam + tuple(grads.get(k) for k in names)


def fused_field(net, xyz, coarse, viewdirs):
    pn.check_trainable(net.engine)
    use_fine = (not coarse) and net.mlp_fine is not None
    mlp = net.mlp_fine if use_fine else net.mlp_coarse
    latent = net.encoder.latent.detach() if net.stop_encoder_grad else net.encoder.latent
    params = [p for _, p in mlp.named_parameters()]
    return _FusedField.apply(net, coarse, xyz, viewdirs, latent, net.poses, net.focal, net.c, *params)
