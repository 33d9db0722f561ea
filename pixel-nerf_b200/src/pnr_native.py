"""
ctypes binding of libpnr_sm90.so (C ABI: include/pnr.h) -- the only way the Python host
code reaches the GPU kernels.  There is no fallback: if the library is missing, or a tensor
is not a contiguous fp32 CUDA tensor, the call raises.

The structures mirror include/pnr.h field for field.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.realpath(__file__))   # realpath: `src/` may be reached through an overlay symlink
LIB_PATH = os.environ.get("PNR_LIB", os.path.join(os.path.dirname(_HERE), "lib", "libpnr_sm90.so"))

PNR_MAX_BLOCKS = 8
ENGINE_AUTO, ENGINE_SIMT, ENGINE_TC, ENGINE_TC_FAST = 0, 1, 2, 4
# "tc_fast": the single-pass fp16 tensor engine (PNR_ENGINE_TC_FAST), inference only; only ever chosen explicitly
ENGINES = {"auto": ENGINE_AUTO, "simt": ENGINE_SIMT, "tc": ENGINE_TC, "tc_fast": ENGINE_TC_FAST}

_fp = C.c_void_p  # device pointers travel as void*


class PnrScene(C.Structure):
    _fields_ = [("latent_nhwc", _fp), ("poses", _fp), ("focal", _fp), ("c", _fp),
                ("n_focal", C.c_int32), ("n_c", C.c_int32), ("SB", C.c_int32), ("NS", C.c_int32),
                ("Hl", C.c_int32), ("Wl", C.c_int32), ("C", C.c_int32),
                ("image_w", C.c_float), ("image_h", C.c_float),
                ("scale_x", C.c_float), ("scale_y", C.c_float),
                ("proj_coarse", _fp), ("proj_fine", _fp)]


class PnrMlp(C.Structure):
    _fields_ = [("d_in", C.c_int32), ("d_latent", C.c_int32), ("d_hidden", C.c_int32),
                ("d_out", C.c_int32), ("n_blocks", C.c_int32), ("combine_layer", C.c_int32),
                ("lin_in_w", _fp), ("lin_in_b", _fp), ("lin_out_w", _fp), ("lin_out_b", _fp),
                ("lin_z_w", _fp * PNR_MAX_BLOCKS), ("lin_z_b", _fp * PNR_MAX_BLOCKS),
                ("fc0_w", _fp * PNR_MAX_BLOCKS), ("fc0_b", _fp * PNR_MAX_BLOCKS),
                ("fc1_w", _fp * PNR_MAX_BLOCKS), ("fc1_b", _fp * PNR_MAX_BLOCKS),
                ("packed", _fp), ("packed_bytes", C.c_size_t)]


class PnrRenderCfg(C.Structure):
    _fields_ = [("n_coarse", C.c_int32), ("n_fine", C.c_int32), ("n_fine_depth", C.c_int32),
                ("depth_std", C.c_float), ("white_bkgd", C.c_int32), ("engine", C.c_int32)]


class PnrNoise(C.Structure):
    _fields_ = [("lin_steps", _fp), ("u_coarse", _fp), ("u_fine", _fp), ("u_fine_jit", _fp),
                ("n_depth", _fp)]


class PnrRenderOut(C.Structure):
    _fields_ = [("rgb_coarse", _fp), ("depth_coarse", _fp), ("weights_coarse", _fp), ("z_coarse", _fp),
                ("rgb_fine", _fp), ("depth_fine", _fp), ("weights_fine", _fp), ("z_fine", _fp)]


class PnrRenderGrad(C.Structure):
    _fields_ = [("d_rgb_coarse", _fp), ("d_depth_coarse", _fp), ("d_weights_coarse", _fp),
                ("d_rgb_fine", _fp), ("d_depth_fine", _fp), ("d_weights_fine", _fp)]


class PnrCameraGrad(C.Structure):
    _fields_ = [("d_poses", _fp), ("d_focal", _fp), ("d_c", _fp)]


class PnrShard(C.Structure):
    _fields_ = [("scene", C.POINTER(PnrScene)), ("mlp_coarse", C.POINTER(PnrMlp)), ("mlp_fine", C.POINTER(PnrMlp)),
                ("noise", C.POINTER(PnrNoise)), ("workspace", _fp), ("workspace_bytes", C.c_size_t),
                ("rays_stage", _fp), ("stage", PnrRenderOut), ("stream", _fp)]


class PnrShardGrad(C.Structure):
    _fields_ = [("rays", _fp), ("z_coarse", _fp), ("z_fine", _fp), ("depth_coarse", _fp), ("up_stage", _fp),
                ("grad_coarse", C.POINTER(PnrMlp)), ("grad_fine", C.POINTER(PnrMlp)), ("d_latent_nhwc", _fp),
                ("arena", _fp), ("arena_count", C.c_int64), ("arena_stage0", _fp),
                ("workspace", _fp), ("workspace_bytes", C.c_size_t), ("stream", _fp)]


class PnrShardCam(C.Structure):
    _fields_ = [("cam", PnrCameraGrad), ("d_rays", _fp)]


POINTS_GRID, POINTS_LATTICE, POINTS_BAND, POINTS_LIST = 1, 2, 3, 4


class PnrPointSource(C.Structure):
    _fields_ = [("kind", C.c_int32), ("lo", C.c_double * 3), ("hi", C.c_double * 3), ("reso", C.c_int32 * 3),
                ("block", C.c_int32), ("apron", C.c_int32), ("n_points", C.c_int64), ("xyz0", _fp),
                ("viewdirs0", _fp)]


class PnrFieldShard(C.Structure):
    _fields_ = [("scene", C.POINTER(PnrScene)), ("mlp", C.POINTER(PnrMlp)), ("plan", _fp), ("plan_bytes", C.c_size_t),
                ("workspace", _fp), ("workspace_bytes", C.c_size_t), ("stream", _fp)]


_lib = None


def declare(L):
    """ctypes signatures of every include/pnr.h entry point on a loaded library handle."""
    L.pnr_abi_version.restype = C.c_int
    L.pnr_last_error.restype = C.c_char_p
    L.pnr_launch_count.restype = C.c_int64
    sz, i32, i64, vp, f32 = C.c_size_t, C.c_int32, C.c_int64, C.c_void_p, C.c_float
    P = C.POINTER
    L.pnr_pack_latent.argtypes = [vp, vp, i32, i32, i32, i32, vp]
    L.pnr_sample_coarse.argtypes = [vp, vp, vp, vp, i64, i32, vp]
    L.pnr_composite.argtypes = [vp, vp, vp, i32, vp, vp, vp, i64, i32, vp]
    L.pnr_gen_rays.argtypes = [vp, i64, i32, i32, f32, f32, f32, f32, f32, f32, i64, i64, vp, vp]
    L.pnr_frames_u8.argtypes = [vp, i64, vp, vp]
    L.pnr_sample_fine.argtypes = [vp, vp, vp, vp, vp, vp, vp, f32, vp, i64, i32, i32, i32, vp]
    L.pnr_field_workspace_bytes.argtypes = [P(PnrScene), P(PnrMlp), i64, i32]
    L.pnr_field_workspace_bytes.restype = sz
    L.pnr_field_eval.argtypes = [P(PnrScene), P(PnrMlp), vp, vp, vp, i64, i32, vp, sz, vp]
    L.pnr_field_backward_workspace_bytes.argtypes = [P(PnrScene), P(PnrMlp), i64]
    L.pnr_field_backward_workspace_bytes.restype = sz
    L.pnr_field_backward.argtypes = [P(PnrScene), P(PnrMlp), vp, vp, vp, P(PnrMlp), vp, vp, i64, vp, sz, vp]
    L.pnr_field_backward.restype = C.c_int
    L.pnr_render_backward_workspace_bytes.argtypes = [P(PnrScene), P(PnrMlp), P(PnrMlp), P(PnrRenderCfg), i64]
    L.pnr_render_backward_workspace_bytes.restype = sz
    L.pnr_render_backward.argtypes = [P(PnrScene), P(PnrMlp), P(PnrMlp), P(PnrRenderCfg), vp, P(PnrNoise),
                                      P(PnrRenderOut), vp, vp, P(PnrMlp), P(PnrMlp), vp, i64, vp, sz, vp]
    L.pnr_render_backward.restype = C.c_int
    L.pnr_render_backward_ex.argtypes = [P(PnrScene), P(PnrMlp), P(PnrMlp), P(PnrRenderCfg), vp, P(PnrNoise),
                                         P(PnrRenderOut), P(PnrRenderGrad), P(PnrMlp), P(PnrMlp), vp, i64, vp, sz, vp]
    L.pnr_render_backward_ex.restype = C.c_int
    L.pnr_field_backward_cam.argtypes = [P(PnrScene), P(PnrMlp), vp, vp, vp, P(PnrMlp), vp, vp, vp, P(PnrCameraGrad),
                                         i64, vp, sz, vp]
    L.pnr_field_backward_cam.restype = C.c_int
    L.pnr_render_backward_cam.argtypes = [P(PnrScene), P(PnrMlp), P(PnrMlp), P(PnrRenderCfg), vp, P(PnrNoise),
                                          P(PnrRenderOut), P(PnrRenderGrad), P(PnrMlp), P(PnrMlp), vp, vp,
                                          P(PnrCameraGrad), i64, vp, sz, vp]
    L.pnr_render_backward_cam.restype = C.c_int
    L.pnr_field_backward_sel.argtypes = L.pnr_field_backward_cam.argtypes
    L.pnr_field_backward_sel.restype = C.c_int
    L.pnr_render_backward_sel.argtypes = L.pnr_render_backward_cam.argtypes
    L.pnr_render_backward_sel.restype = C.c_int
    L.pnr_gen_rays_backward.argtypes = [vp, vp, i64, i32, i32, f32, f32, f32, f32, i64, i64, vp, vp]
    L.pnr_gen_rays_backward.restype = C.c_int
    L.pnr_composite_backward.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, vp, i64, i32, vp]
    L.pnr_composite_backward.restype = C.c_int
    L.pnr_render_workspace_bytes.argtypes = [P(PnrScene), P(PnrMlp), P(PnrMlp), P(PnrRenderCfg), i64]
    L.pnr_render_workspace_bytes.restype = sz
    L.pnr_render.argtypes = [P(PnrScene), P(PnrMlp), P(PnrMlp), P(PnrRenderCfg), vp, P(PnrNoise),
                             P(PnrRenderOut), i64, vp, sz, vp]
    L.pnr_pack_mlp_bytes.argtypes = [P(PnrMlp)]
    L.pnr_pack_mlp_bytes.restype = sz
    L.pnr_pack_mlp.argtypes = [P(PnrMlp), vp, sz, vp]
    L.pnr_project_latent_bytes.argtypes = [P(PnrScene), P(PnrMlp)]
    L.pnr_project_latent_bytes.restype = sz
    L.pnr_project_latent.argtypes = [P(PnrScene), P(PnrMlp), vp, sz, vp, sz, vp]
    if hasattr(L, "pnr_mgpu_create"):     # (the host-emulator build of tests/cuda_emu has no multi-GPU driver)
        L.pnr_mgpu_create.argtypes = [P(i32), i32, P(vp)]
        L.pnr_mgpu_destroy.argtypes = [vp]
        L.pnr_mgpu_size.argtypes = [vp]
        L.pnr_mgpu_size.restype = i32
        L.pnr_mgpu_peer_store.argtypes = [vp, i32]
        L.pnr_mgpu_peer_store.restype = i32
        L.pnr_mgpu_broadcast.argtypes = [vp, vp, P(vp), sz, P(vp)]
        L.pnr_mgpu_render.argtypes = [vp, P(PnrShard), P(PnrRenderCfg), vp, P(PnrRenderOut), i64, vp]
        L.pnr_mgpu_peer_load.argtypes = [vp, i32]
        L.pnr_mgpu_peer_load.restype = i32
        L.pnr_mgpu_render_backward.argtypes = [vp, P(PnrShard), P(PnrShardGrad), P(PnrRenderCfg), P(PnrRenderGrad),
                                               P(PnrMlp), P(PnrMlp), vp, i64, vp]
        L.pnr_mgpu_render_backward_cam.argtypes = [vp, P(PnrShard), P(PnrShardGrad), P(PnrShardCam), P(PnrRenderCfg),
                                                   P(PnrRenderGrad), P(PnrMlp), P(PnrMlp), vp, vp, P(PnrCameraGrad),
                                                   i64, vp]
        L.pnr_mgpu_render_backward_sel.argtypes = L.pnr_mgpu_render_backward_cam.argtypes
        L.pnr_sum_into.argtypes = [vp, P(vp), i32, i64, vp]
        for name in ("pnr_mgpu_create", "pnr_mgpu_destroy", "pnr_mgpu_broadcast", "pnr_mgpu_render",
                     "pnr_mgpu_render_backward", "pnr_mgpu_render_backward_cam", "pnr_mgpu_render_backward_sel",
                     "pnr_sum_into"):
            getattr(L, name).restype = C.c_int
    if hasattr(L, "pnr_mgpu_field_eval"):  # (the host-emulator builds of tests/cuda_emu have it only with mesh extraction)
        L.pnr_mgpu_field_workspace_bytes.argtypes = [P(PnrScene), P(PnrMlp), i64, i32]
        L.pnr_mgpu_field_workspace_bytes.restype = sz
        L.pnr_mgpu_field_eval.argtypes = [vp, P(PnrFieldShard), P(PnrPointSource), i64, i64, i32, i32, i32, vp, vp]
        L.pnr_mgpu_field_eval.restype = C.c_int
    if hasattr(L, "pnr_grid_points"):     # (the host-emulator build of tests/cuda_emu has no mesh extraction)
        f64 = C.c_double
        L.pnr_grid_points.argtypes = [P(f64), P(f64), P(i32), i64, i64, vp, vp, vp]
        L.pnr_mc_workspace_bytes.argtypes = [i32, i32, i32]
        L.pnr_mc_workspace_bytes.restype = sz
        L.pnr_mc_count.argtypes = [vp, i32, i32, i32, f64, vp, vp, sz, vp]
        L.pnr_mc_emit.argtypes = [vp, i32, i32, i32, f64, vp, vp, i64, i64, vp, sz, vp]
        L.pnr_mc_vertex_attrs.argtypes = [vp, i32, i32, i32, f64, P(f64), P(f64), vp, vp, vp, i64, vp, sz, vp]
        for name in ("pnr_grid_points", "pnr_mc_count", "pnr_mc_emit", "pnr_mc_vertex_attrs"):
            getattr(L, name).restype = C.c_int
        L.pnr_band_plan_bytes.argtypes = [P(i32), i32, i32]
        L.pnr_band_plan_bytes.restype = sz
        L.pnr_band_lattice_points.argtypes = [P(f64), P(f64), P(i32), i32, i64, i64, vp, vp, vp]
        L.pnr_band_plan.argtypes = [vp, P(i32), i32, f64, i32, vp, vp, sz, vp]
        L.pnr_band_points.argtypes = [P(f64), P(f64), P(i32), i32, i32, vp, sz, i64, i64, i64, vp, vp, vp]
        L.pnr_band_mc_workspace_bytes.argtypes = [i64]
        L.pnr_band_mc_workspace_bytes.restype = sz
        L.pnr_band_mc_count.argtypes = [vp, i64, P(i32), i32, i32, f64, vp, sz, vp, vp, sz, vp]
        L.pnr_band_mc_emit.argtypes = [vp, i64, P(i32), i32, i32, f64, vp, sz, vp, vp, i64, i64, vp, sz, vp]
        L.pnr_band_mc_vertex_attrs.argtypes = [vp, i64, P(i32), i32, i32, f64, P(f64), P(f64), vp, sz, vp, vp, vp, i64,
                                               vp, sz, vp]
        L.pnr_tsdf_fuse.argtypes = [vp, vp, i32, i32, i32, vp, f32, f32, f32, f32, P(f64), P(f64), P(i32), f64, f64,
                                    vp, vp]
        L.pnr_paint_vertices.argtypes = [vp, vp, i64, vp, vp, vp, i32, i32, i32, vp, f32, f32, f32, f32, f64, f64, f64,
                                         vp, vp, vp]
        for name in ("pnr_band_lattice_points", "pnr_band_plan", "pnr_band_points", "pnr_band_mc_count",
                     "pnr_band_mc_emit", "pnr_band_mc_vertex_attrs", "pnr_tsdf_fuse", "pnr_paint_vertices"):
            getattr(L, name).restype = C.c_int
    if hasattr(L, "pnr_mesh_components"):  # (not in the host-emulator builds without csrc/pnr_mesh.cu)
        L.pnr_mesh_workspace_bytes.argtypes = [i64, i64]
        L.pnr_mesh_workspace_bytes.restype = sz
        L.pnr_mesh_components.argtypes = [vp, i64, i64, vp, vp, P(i64), vp, sz, vp]
        L.pnr_mesh_compact_count.argtypes = [vp, i64, i64, vp, vp, vp, vp, sz, vp]
        L.pnr_mesh_compact_emit.argtypes = [vp, i64, i64, vp, vp, i64, i64, vp, sz, vp]
        for name in ("pnr_mesh_components", "pnr_mesh_compact_count", "pnr_mesh_compact_emit"):
            getattr(L, name).restype = C.c_int
        L.pnr_decimate_workspace_bytes.argtypes = [i64, i64]
        L.pnr_decimate_workspace_bytes.restype = sz
        L.pnr_decimate_init.argtypes = [vp, i64, vp, i64, vp, vp, vp, sz, vp]
        L.pnr_decimate_select.argtypes = [vp, i64, vp, i64, vp, vp, C.c_double, vp, vp, vp, P(i64), vp, sz, vp]
        L.pnr_decimate_apply.argtypes = [vp, i64, i64, vp, vp, i64, vp, vp, P(i64), vp, sz, vp]
        for name in ("pnr_decimate_init", "pnr_decimate_select", "pnr_decimate_apply"):
            getattr(L, name).restype = C.c_int
    L.pnr_set_deterministic.argtypes = [C.c_int]
    L.pnr_set_deterministic.restype = C.c_int
    L.pnr_get_deterministic.restype = C.c_int
    if hasattr(L, "pnr_upsample_bilinear_ac_backward"):   # (not in the host-emulator build of tests/cuda_emu)
        L.pnr_upsample_bilinear_ac_backward.argtypes = [vp, i64, i32, i32, i32, i32, i32, vp, vp]
        L.pnr_upsample_bilinear_ac_backward.restype = C.c_int
    L.pnr_gemm_nt.argtypes = [vp, i32, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp]
    L.pnr_gemm_nt.restype = C.c_int
    L.pnr_profile_begin.restype = C.c_int
    L.pnr_tc_status.argtypes = [P(C.c_int)]
    L.pnr_tc_status.restype = C.c_int
    L.pnr_profile_end.argtypes = [P(C.c_double), P(C.c_int64)]
    L.pnr_profile_end.restype = C.c_int
    for name in ("pnr_pack_latent", "pnr_sample_coarse", "pnr_composite", "pnr_sample_fine",
                 "pnr_field_eval", "pnr_render", "pnr_pack_mlp", "pnr_project_latent", "pnr_gen_rays",
                 "pnr_frames_u8"):
        getattr(L, name).restype = C.c_int
    return L


def lib():
    """Loads the shared library once; raises (never falls back) if it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"libpnr_sm90.so not found at {LIB_PATH}: build it with `python -c 'import __graft_entry__ as g; "
            "g.build()'` (or `make -C pixel-nerf_b200/csrc`). There is no CPU fallback for the render path.")
    L = declare(C.CDLL(LIB_PATH))
    if L.pnr_abi_version() != 2:
        raise RuntimeError("libpnr_sm90.so ABI version mismatch")
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise RuntimeError(f"libpnr_sm90 error {rc}: {lib().pnr_last_error().decode()}")


def check_trainable(engine):
    """Raises for an engine whose forward the fused backward cannot reproduce ("tc_fast": its backward would
    differentiate the exact engine's forward instead), before a grad-mode node runs that forward."""
    if engine == "tc_fast":
        raise RuntimeError('engine "tc_fast" is inference only: the single-pass fp16 forward has no matching backward; '
                           'training needs net.engine = "tc" or "auto" (or run this call under torch.no_grad())')


def sync_deterministic():
    """Sets the library's deterministic-mode flag of the calling thread from torch.are_deterministic_algorithms_enabled()
    (warn_only counts as on) and returns it.  Call it in the thread that makes the library call, before its workspace
    query: the flag is thread-local and autograd runs backward on its own thread."""
    on = torch.are_deterministic_algorithms_enabled()
    lib().pnr_set_deterministic(1 if on else 0)
    return on


def upsample_bilinear_ac_backward(d_out, in_hw):
    """pnr_upsample_bilinear_ac_backward: gradient [N][C][h_in][w_in] of F.interpolate(x, d_out's size,
    mode="bilinear", align_corners=True) from d_out, in a fixed summation order."""
    d_out = d_out.to(torch.float32).contiguous()
    N, Cc, h_out, w_out = d_out.shape
    d_in = torch.empty(N, Cc, int(in_hw[0]), int(in_hw[1]), dtype=torch.float32, device=d_out.device)
    with torch.cuda.device(d_out.device):
        check(lib().pnr_upsample_bilinear_ac_backward(dptr(d_out, "d_out"), N, Cc, d_in.shape[2], d_in.shape[3], h_out,
                                                      w_out, dptr(d_in), stream_ptr(d_out.device)))
    return d_in


def dptr(t, name="tensor"):
    """Device pointer of a contiguous fp32 CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
        raise RuntimeError(f"{name}: expected a contiguous float32 CUDA tensor, got "
                           f"{t.dtype} on {t.device} (contiguous={t.is_contiguous()}); "
                           "the fused render path has no CPU fallback")
    return C.c_void_p(t.data_ptr())


def stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def gen_rays(poses, width, height, fx, fy, cx, cy, z_near, z_far, first=0, count=None, out=None):
    """pnr_gen_rays: rays [count][8] of pixels [first, first+count) of the (NV,H,W) grid of `poses` (NV,4,4) c2w."""
    nv = poses.shape[0]
    total = nv * width * height
    if count is None:
        count = total - first
    poses = poses.to(torch.float32).contiguous()
    if out is None:
        out = torch.empty(count, 8, device=poses.device, dtype=torch.float32)
    elif out.shape != (count, 8):
        raise RuntimeError(f"gen_rays: out has shape {tuple(out.shape)}, expected {(count, 8)}")
    with torch.cuda.device(poses.device):
        check(lib().pnr_gen_rays(dptr(poses, "poses"), nv, int(width), int(height), float(fx), float(fy), float(cx),
                                 float(cy), float(z_near), float(z_far), int(first), int(count), dptr(out, "rays"),
                                 stream_ptr(poses.device)))
    return out


class _GenRays(torch.autograd.Function):
    """gen_rays with a gradient w.r.t. the camera-to-world poses: forward pnr_gen_rays, backward pnr_gen_rays_backward."""

    @staticmethod
    def forward(ctx, poses, width, height, fx, fy, cx, cy, z_near, z_far):
        ctx.args = (poses.shape, poses.dtype, int(width), int(height), float(fx), float(fy), float(cx), float(cy))
        p = poses.detach().to(torch.float32).contiguous()
        ctx.save_for_backward(p)
        return gen_rays(p, width, height, fx, fy, cx, cy, z_near, z_far)

    @staticmethod
    def backward(ctx, d_rays):
        shape, dtype, W, H, fx, fy, cx, cy = ctx.args
        (p,) = ctx.saved_tensors
        d_rays = d_rays.to(torch.float32).contiguous()
        d_poses = torch.zeros(p.shape, dtype=torch.float32, device=p.device)
        with torch.cuda.device(p.device):
            check(lib().pnr_gen_rays_backward(dptr(d_rays, "d_rays"), dptr(p, "poses"), p.shape[0], W, H, fx, fy, cx,
                                              cy, 0, d_rays.shape[0], dptr(d_poses), stream_ptr(p.device)))
        return (d_poses.to(dtype),) + (None,) * 8


def gen_rays_autograd(poses, width, height, fx, fy, cx, cy, z_near, z_far):
    """gen_rays of every pixel as an autograd node on `poses` (the same bits as gen_rays)."""
    return _GenRays.apply(poses, width, height, fx, fy, cx, cy, z_near, z_far)


def frames_u8(rgb, out=None):
    """pnr_frames_u8: (rgb * 255).astype(uint8) of a float32 CUDA tensor, same shape."""
    rgb = rgb.contiguous()
    if out is None:
        out = torch.empty(rgb.shape, device=rgb.device, dtype=torch.uint8)
    elif not (out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous() and out.numel() == rgb.numel()):
        raise RuntimeError("frames_u8: out must be a contiguous uint8 CUDA tensor with as many elements as rgb")
    with torch.cuda.device(rgb.device):
        check(lib().pnr_frames_u8(dptr(rgb, "rgb"), rgb.numel(), C.c_void_p(out.data_ptr()), stream_ptr(rgb.device)))
    return out


def grid_points(lo, hi, reso, first, count, xyz, viewdirs=None):
    """pnr_grid_points: points [first, first+count) of util.gen_grid(*zip(lo, hi, reso), ij_indexing=True) into
    xyz [>= count, 3] (and -p/|p| into viewdirs), both contiguous fp32 CUDA tensors."""
    for t, name in ((xyz, "xyz"), (viewdirs, "viewdirs")):
        if t is not None and (t.dim() != 2 or t.shape[0] < count or t.shape[1] != 3):
            raise RuntimeError(f"grid_points: {name} must be [>= {count}, 3], got {tuple(t.shape)}")
    dev = xyz.device
    with torch.cuda.device(dev):
        check(lib().pnr_grid_points((C.c_double * 3)(*map(float, lo)), (C.c_double * 3)(*map(float, hi)),
                                    (C.c_int32 * 3)(*map(int, reso)), int(first), int(count), dptr(xyz, "xyz"),
                                    dptr(viewdirs, "viewdirs"), stream_ptr(dev)))


def marching_cubes(vol, iso, *, bounds=None):
    """pnr_mc_count + pnr_mc_emit on a contiguous fp32 CUDA volume (nx, ny, nz) -> (vertices float64 [N, 3] in grid
    index space, triangles int64 [M, 3]), CUDA tensors on vol's device.  Synchronises once, to size the outputs.
    With bounds = (lo, hi), the world box the grid spans, pnr_mc_vertex_attrs also runs and the result is
    (vertices, triangles, normals float64 [N, 3], xyz float32 [N, 3], viewdirs float32 [N, 3])."""
    if vol.dim() != 3:
        raise RuntimeError(f"marching_cubes: expected a 3-D volume, got shape {tuple(vol.shape)}")
    nx, ny, nz = vol.shape
    dev = vol.device
    L = lib()
    ws = torch.empty(max(int(L.pnr_mc_workspace_bytes(nx, ny, nz)), 1), dtype=torch.uint8, device=dev)
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        s = stream_ptr(dev)
        check(L.pnr_mc_count(dptr(vol, "vol"), nx, ny, nz, float(iso), C.c_void_p(counts.data_ptr()),
                             C.c_void_p(ws.data_ptr()), ws.numel(), s))
        nv, nt = counts.tolist()
        verts = torch.empty(nv, 3, dtype=torch.float64, device=dev)
        tris = torch.empty(nt, 3, dtype=torch.int64, device=dev)
        check(L.pnr_mc_emit(dptr(vol, "vol"), nx, ny, nz, float(iso), C.c_void_p(verts.data_ptr()),
                            C.c_void_p(tris.data_ptr()), nv, nt, C.c_void_p(ws.data_ptr()), ws.numel(), s))
        if bounds is None:
            return verts, tris
        lo, hi = bounds
        normals = torch.empty(nv, 3, dtype=torch.float64, device=dev)
        xyz = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        viewdirs = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        check(L.pnr_mc_vertex_attrs(dptr(vol, "vol"), nx, ny, nz, float(iso), (C.c_double * 3)(*map(float, lo)),
                                    (C.c_double * 3)(*map(float, hi)), C.c_void_p(normals.data_ptr()), dptr(xyz),
                                    dptr(viewdirs), nv, C.c_void_p(ws.data_ptr()), ws.numel(), s))
    return verts, tris, normals, xyz, viewdirs


def tsdf_fuse(depth, opacity, poses, fx, fy, cx, cy, lo, hi, reso, trunc, min_opacity):
    """pnr_tsdf_fuse: depth and opacity maps [V, H, W] and camera-to-world poses [V, 4, 4] (fp32 CUDA tensors on one
    device) -> the fused TSDF [nx, ny, nz] fp32 on that device, positive outside (rule: include/pnr.h)."""
    if depth.dim() != 3 or opacity.shape != depth.shape:
        raise RuntimeError(f"tsdf_fuse: depth and opacity must both be [V, H, W], got {tuple(depth.shape)} and "
                           f"{tuple(opacity.shape)}")
    V, H, W = depth.shape
    if tuple(poses.shape) != (V, 4, 4):
        raise RuntimeError(f"tsdf_fuse: poses must be [{V}, 4, 4], got {tuple(poses.shape)}")
    dev = depth.device
    if opacity.device != dev or poses.device != dev:
        raise RuntimeError(f"tsdf_fuse: depth, opacity and poses must be on one device, got {dev}, {opacity.device} "
                           f"and {poses.device}")
    reso = [int(r) for r in reso]
    tsdf = torch.empty(*reso, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        check(lib().pnr_tsdf_fuse(dptr(depth, "depth"), dptr(opacity, "opacity"), V, W, H, dptr(poses, "poses"),
                                  float(fx), float(fy), float(cx), float(cy), *_bounds3(lo, hi), _reso3(reso),
                                  float(trunc), float(min_opacity), dptr(tsdf), stream_ptr(dev)))
    return tsdf


def paint_vertices(xyz, normals, rgb, depth, opacity, poses, fx, fy, cx, cy, trunc, min_opacity, background):
    """pnr_paint_vertices: world-space vertices and unit outward normals [n, 3] float64, rendered maps rgb [V, H, W, 3],
    depth and opacity [V, H, W] and camera-to-world poses [V, 4, 4] (fp32), all CUDA tensors on one device -> (rgb
    [n, 3] fp32, weight [n] float64) on that device: the cos-weighted mean of the pixels of the views that see each
    vertex, NaN and 0 where none does (rule: include/pnr.h)."""
    if depth.dim() != 3 or opacity.shape != depth.shape:
        raise RuntimeError(f"paint_vertices: depth and opacity must both be [V, H, W], got {tuple(depth.shape)} and "
                           f"{tuple(opacity.shape)}")
    V, H, W = depth.shape
    if tuple(rgb.shape) != (V, H, W, 3):
        raise RuntimeError(f"paint_vertices: rgb must be [{V}, {H}, {W}, 3], got {tuple(rgb.shape)}")
    if tuple(poses.shape) != (V, 4, 4):
        raise RuntimeError(f"paint_vertices: poses must be [{V}, 4, 4], got {tuple(poses.shape)}")
    if xyz.dim() != 2 or xyz.shape[1] != 3 or normals.shape != xyz.shape:
        raise RuntimeError(f"paint_vertices: xyz and normals must both be [n, 3], got {tuple(xyz.shape)} and "
                           f"{tuple(normals.shape)}")
    dev = depth.device
    for t, name in ((xyz, "xyz"), (normals, "normals"), (rgb, "rgb"), (opacity, "opacity"), (poses, "poses")):
        if t.device != dev:
            raise RuntimeError(f"paint_vertices: {name} is on {t.device}, the maps on {dev}")
    for t, name in ((xyz, "xyz"), (normals, "normals")):
        if not (t.dtype == torch.float64 and t.is_contiguous()):
            raise RuntimeError(f"paint_vertices: {name} must be a contiguous float64 tensor, got {t.dtype} "
                               f"(contiguous={t.is_contiguous()})")
    n = xyz.shape[0]
    out = torch.empty(n, 3, dtype=torch.float32, device=dev)
    weight = torch.empty(n, dtype=torch.float64, device=dev)
    if n == 0:
        return out, weight
    with torch.cuda.device(dev):
        check(lib().pnr_paint_vertices(C.c_void_p(xyz.data_ptr()), C.c_void_p(normals.data_ptr()), n,
                                       dptr(rgb, "rgb"), dptr(depth, "depth"), dptr(opacity, "opacity"), V, W, H,
                                       dptr(poses, "poses"), float(fx), float(fy), float(cx), float(cy), float(trunc),
                                       float(min_opacity), float(background), dptr(out),
                                       C.c_void_p(weight.data_ptr()), stream_ptr(dev)))
    return out, weight


def _mesh_tris(tris, n_verts):
    if tris.dim() != 2 or tris.shape[1] != 3 or tris.dtype != torch.int64 or not tris.is_cuda:
        raise RuntimeError(f"mesh: tris must be an int64 CUDA tensor [M, 3], got {tris.dtype} {tuple(tris.shape)} on "
                           f"{tris.device}")
    if int(n_verts) < 0:
        raise RuntimeError(f"mesh: n_verts must be >= 0, got {n_verts}")
    return tris.contiguous()


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t.numel() else None


def mesh_components(tris, n_verts):
    """pnr_mesh_components on an int64 CUDA tensor tris [M, 3] of vertex ids in [0, n_verts) -> (label [n_verts]
    int64: the smallest vertex id of each vertex's component, tri_count [n_verts] int64: each component's triangles
    at its label, 0 elsewhere, the number of components with a triangle), on tris' device.  Synchronises once.
    Raises ValueError for an id outside [0, n_verts) (rule: include/pnr.h)."""
    tris = _mesh_tris(tris, n_verts)
    n, m, dev = int(n_verts), tris.shape[0], tris.device
    L = lib()
    ws = torch.empty(max(int(L.pnr_mesh_workspace_bytes(n, m)), 1), dtype=torch.uint8, device=dev)
    label = torch.empty(n, dtype=torch.int64, device=dev)
    tri_count = torch.empty(n, dtype=torch.int64, device=dev)
    count = C.c_int64(0)
    with torch.cuda.device(dev):
        rc = L.pnr_mesh_components(_ptr(tris), m, n, _ptr(label), _ptr(tri_count), C.byref(count),
                                   C.c_void_p(ws.data_ptr()), ws.numel(), stream_ptr(dev))
    if rc == -1 and b"outside [0, n_verts)" in L.pnr_last_error():
        raise ValueError(f"triangles use a vertex id outside [0, {n})")
    check(rc)
    return label, tri_count, count.value


def mesh_compact(tris, n_verts, label, keep_root):
    """pnr_mesh_compact_count + pnr_mesh_compact_emit: the vertices whose root (label) has keep_root [n_verts] uint8
    set, and the triangles among them -> (vert_ids [K] int64: their old ids ascending, tris [T, 3] int64 through the
    new ids), on tris' device.  Synchronises once, to size the outputs."""
    tris = _mesh_tris(tris, n_verts)
    n, m, dev = int(n_verts), tris.shape[0], tris.device
    if tuple(label.shape) != (n,) or label.dtype != torch.int64 or label.device != dev:
        raise RuntimeError(f"mesh_compact: label must be int64 [{n}] on {dev}")
    if tuple(keep_root.shape) != (n,) or keep_root.dtype != torch.uint8 or keep_root.device != dev:
        raise RuntimeError(f"mesh_compact: keep_root must be uint8 [{n}] on {dev}")
    label, keep_root = label.contiguous(), keep_root.contiguous()
    L = lib()
    ws = torch.empty(max(int(L.pnr_mesh_workspace_bytes(n, m)), 1), dtype=torch.uint8, device=dev)
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        s = stream_ptr(dev)
        check(L.pnr_mesh_compact_count(_ptr(tris), m, n, _ptr(label), _ptr(keep_root), C.c_void_p(counts.data_ptr()),
                                       C.c_void_p(ws.data_ptr()), ws.numel(), s))
        nv, nt = counts.tolist()
        vert_ids = torch.empty(nv, dtype=torch.int64, device=dev)
        tris_out = torch.empty(nt, 3, dtype=torch.int64, device=dev)
        check(L.pnr_mesh_compact_emit(_ptr(tris), m, n, _ptr(vert_ids), _ptr(tris_out), nv, nt,
                                      C.c_void_p(ws.data_ptr()), ws.numel(), s))
    return vert_ids, tris_out


class Decimator:
    """The state of one pnr_decimate_* run on a mesh's device: xyz [N, 3] float64, tris [M, 3] int64 (ids checked in
    [0, N) on the device: ValueError otherwise), the quadrics [N, 10] float64 and a workspace sized for (N, M).
    select() -> (c, d, err) of one round's selected collapses, ascending c, and whether max_error held some back;
    apply(c, d) collapses them and returns the new triangle count (rule: include/pnr.h).  Each call synchronises once.
    The rounds ping-pong between tris and a second buffer, so tris is overwritten: pass a tensor the caller owns."""

    def __init__(self, xyz, tris):
        tris = _mesh_tris(tris, xyz.shape[0])
        if xyz.dim() != 2 or xyz.shape[1] != 3 or xyz.dtype != torch.float64 or xyz.device != tris.device:
            raise RuntimeError(f"decimate: xyz must be float64 [N, 3] on {tris.device}")
        self.xyz, self.tris, self.dev = xyz.contiguous(), tris, tris.device
        self.n = n = xyz.shape[0]
        L = self.L = lib()
        self.ws = torch.empty(max(int(L.pnr_decimate_workspace_bytes(n, tris.shape[0])), 1), dtype=torch.uint8,
                              device=self.dev)
        self.quadrics = torch.empty(n, 10, dtype=torch.float64, device=self.dev)
        self.frozen = torch.empty(n, dtype=torch.uint8, device=self.dev)
        self.spare = torch.empty_like(tris)
        with torch.cuda.device(self.dev):
            rc = L.pnr_decimate_init(_ptr(self.xyz), n, _ptr(tris), tris.shape[0], _ptr(self.quadrics),
                                     _ptr(self.frozen), C.c_void_p(self.ws.data_ptr()), self.ws.numel(),
                                     stream_ptr(self.dev))
        if rc == -1 and b"outside [0, n_verts)" in L.pnr_last_error():
            raise ValueError(f"triangles use a vertex id outside [0, {n})")
        check(rc)

    def select(self, max_error=None):
        bound = float("inf") if max_error is None else float(max_error)
        k = max(self.n // 2, 1)                  # (never 0, so that no output is NULL for a 1-vertex mesh)
        c, d = (torch.empty(k, dtype=torch.int64, device=self.dev) for _ in range(2))
        err = torch.empty(k, dtype=torch.float64, device=self.dev)
        counts = (C.c_int64 * 2)()
        with torch.cuda.device(self.dev):
            check(self.L.pnr_decimate_select(_ptr(self.xyz), self.n, _ptr(self.tris), self.tris.shape[0],
                                             _ptr(self.quadrics), _ptr(self.frozen), bound, _ptr(c), _ptr(d), _ptr(err),
                                             C.cast(counts, C.POINTER(C.c_int64)), C.c_void_p(self.ws.data_ptr()),
                                             self.ws.numel(), stream_ptr(self.dev)))
        k = counts[0]
        return c[:k], d[:k], err[:k], bool(counts[1])

    def apply(self, c, d):
        c, d = c.contiguous(), d.contiguous()
        m = self.tris.shape[0]
        count = C.c_int64(0)
        with torch.cuda.device(self.dev):
            check(self.L.pnr_decimate_apply(_ptr(self.tris), m, self.n, _ptr(c), _ptr(d), c.numel(),
                                            _ptr(self.quadrics), _ptr(self.spare), C.byref(count),
                                            C.c_void_p(self.ws.data_ptr()), self.ws.numel(), stream_ptr(self.dev)))
        self.tris, self.spare = self.spare[:count.value], self.tris
        return count.value


BAND_MAX_BLOCK = 256


def _reso3(reso):
    return (C.c_int32 * 3)(*map(int, reso))


def _bounds3(lo, hi):
    return (C.c_double * 3)(*map(float, lo)), (C.c_double * 3)(*map(float, hi))


def band_lattice_size(reso, block):
    """Points of the narrow band's coarse lattice: the grid indices min(j * block, n - 1), j = 0 .. ceil((n - 1) /
    block), per axis."""
    m = [(int(n) - 1 + block - 1) // block + 1 for n in reso]
    return m[0] * m[1] * m[2]


def band_lattice_points(lo, hi, reso, block, first, count, xyz, viewdirs=None):
    """pnr_band_lattice_points: lattice points [first, first+count) into xyz / viewdirs, as grid_points writes them."""
    dev = xyz.device
    with torch.cuda.device(dev):
        check(lib().pnr_band_lattice_points(*_bounds3(lo, hi), _reso3(reso), int(block), int(first), int(count),
                                            dptr(xyz, "xyz"), dptr(viewdirs, "viewdirs"), stream_ptr(dev)))


class BandPlan:
    """pnr_band_plan's result: the plan buffer (a CUDA byte tensor) and its counts."""

    def __init__(self, reso, block, apron, buf, n_active, n_points):
        self.reso, self.block, self.apron, self.buf = reso, block, apron, buf
        self.n_active, self.n_points = n_active, n_points

    def args(self):
        return _reso3(self.reso), self.block, int(self.apron)


def band_plan(coarse, reso, block, iso, apron=False):
    """pnr_band_plan on the lattice's fp32 CUDA sigma (band_lattice_size(reso, block) values) -> BandPlan.
    Synchronises once, to read the active-block and refinement-point counts."""
    reso, block = [int(r) for r in reso], int(block)
    dev = coarse.device
    L = lib()
    nbytes = int(L.pnr_band_plan_bytes(_reso3(reso), block, int(bool(apron))))
    if nbytes == 0:
        raise RuntimeError(f"band_plan: invalid grid {reso} or block {block}")
    if coarse.numel() != band_lattice_size(reso, block):
        raise RuntimeError(f"band_plan: coarse sigma has {coarse.numel()} values, the lattice "
                           f"{band_lattice_size(reso, block)}")
    buf = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        check(L.pnr_band_plan(dptr(coarse, "coarse"), _reso3(reso), block, float(iso), int(bool(apron)),
                              C.c_void_p(counts.data_ptr()), C.c_void_p(buf.data_ptr()), nbytes, stream_ptr(dev)))
        n_active, n_points = counts.tolist()
    return BandPlan(reso, block, bool(apron), buf, n_active, n_points)


def band_points(plan, lo, hi, first, count, xyz, viewdirs=None):
    """pnr_band_points: refinement points [first, first+count) of `plan` into xyz / viewdirs."""
    dev = xyz.device
    with torch.cuda.device(dev):
        check(lib().pnr_band_points(*_bounds3(lo, hi), *plan.args(), C.c_void_p(plan.buf.data_ptr()), plan.buf.numel(),
                                    plan.n_points, int(first), int(count), dptr(xyz, "xyz"),
                                    dptr(viewdirs, "viewdirs"), stream_ptr(dev)))


def band_marching_cubes(sigma, plan, iso, *, bounds=None):
    """pnr_band_mc_count + pnr_band_mc_emit on the fp32 CUDA sigma of plan's refinement points, in their order ->
    (vertices float64 [N, 3] in grid index space, triangles int64 [M, 3]), as marching_cubes returns them.
    Synchronises once, to size the outputs.  With bounds = (lo, hi), pnr_band_mc_vertex_attrs also runs (the plan
    must have been made with apron) and the result is (vertices, triangles, normals, xyz, viewdirs)."""
    if sigma.numel() != plan.n_points:
        raise RuntimeError(f"band_marching_cubes: sigma has {sigma.numel()} values, the plan {plan.n_points} points")
    if bounds is not None and not plan.apron:
        raise RuntimeError("band_marching_cubes: vertex attributes need a plan made with apron=True")
    dev = sigma.device
    L = lib()
    M = plan.n_points
    ws = torch.empty(max(int(L.pnr_band_mc_workspace_bytes(M)), 1), dtype=torch.uint8, device=dev)
    pp = (C.c_void_p(plan.buf.data_ptr()), plan.buf.numel())
    head = (dptr(sigma, "sigma"), M, *plan.args(), float(iso))
    tail = (C.c_void_p(ws.data_ptr()), ws.numel())
    counts = torch.empty(2, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        s = stream_ptr(dev)
        check(L.pnr_band_mc_count(*head, *pp, C.c_void_p(counts.data_ptr()), *tail, s))
        nv, nt = counts.tolist()
        verts = torch.empty(nv, 3, dtype=torch.float64, device=dev)
        tris = torch.empty(nt, 3, dtype=torch.int64, device=dev)
        check(L.pnr_band_mc_emit(*head, *pp, C.c_void_p(verts.data_ptr()), C.c_void_p(tris.data_ptr()), nv, nt,
                                 *tail, s))
        if bounds is None:
            return verts, tris
        normals = torch.empty(nv, 3, dtype=torch.float64, device=dev)
        xyz = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        viewdirs = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        check(L.pnr_band_mc_vertex_attrs(*head, *_bounds3(*bounds), *pp, C.c_void_p(normals.data_ptr()), dptr(xyz),
                                         dptr(viewdirs), nv, *tail, s))
    return verts, tris, normals, xyz, viewdirs


def point_source(kind, lo=(0.0, 0.0, 0.0), hi=(0.0, 0.0, 0.0), reso=(1, 1, 1), block=0, apron=False, n_points=0,
                 xyz0=None, viewdirs0=None):
    """PnrPointSource for pnr_mgpu_field_eval: POINTS_GRID (lo, hi, reso), POINTS_LATTICE (+ block), POINTS_BAND
    (+ apron and the plan's n_points) or POINTS_LIST (xyz0 / viewdirs0 [count, 3] fp32 CUDA tensors on gpus[0])."""
    s = PnrPointSource()
    s.kind = int(kind)
    s.lo[:], s.hi[:], s.reso[:] = [float(v) for v in lo], [float(v) for v in hi], [int(r) for r in reso]
    s.block, s.apron, s.n_points = int(block), int(bool(apron)), int(n_points)
    s.xyz0, s.viewdirs0 = dptr(xyz0, "xyz0"), dptr(viewdirs0, "viewdirs0")
    return s


def mgpu_field_eval(handle, shards, src, count, chunk, engine, channel, out0):
    """pnr_mgpu_field_eval: channels [channel, channel + out0.shape[1]) of the field at the source's points [0, count),
    in chunks of `chunk` points sharded over the handle's devices -> out0 [count, n_channels] (fp32 CUDA, gpus[0]),
    ordered on out0's device's current stream.  shards: a PnrFieldShard array, one per device of the handle."""
    dev = out0.device
    with torch.cuda.device(dev):
        check(lib().pnr_mgpu_field_eval(handle, shards, C.byref(src), int(count), int(chunk), int(engine), int(channel),
                                        int(out0.shape[1]), dptr(out0, "out0"), stream_ptr(dev)))
    return out0


def profile_begin():
    check(lib().pnr_profile_begin())


def profile_end():
    """-> (total device ms of the dominant kernel, launches) since profile_begin()."""
    ms, n = C.c_double(0.0), C.c_int64(0)
    check(lib().pnr_profile_end(C.byref(ms), C.byref(n)))
    return ms.value, n.value


def tc_status():
    """Synchronise and return the tensor engine's status word (0 = ok)."""
    v = C.c_int(0)
    check(lib().pnr_tc_status(C.byref(v)))
    return v.value


def tc_counters():
    arr = (C.c_ulonglong * 8)()
    lib().pnr_tc_counters.restype = C.c_int
    check(lib().pnr_tc_counters(arr))
    return list(arr)


def launch_count():
    return int(lib().pnr_launch_count())


# ------------------------------------------------------------------------------------------
# Workspace cache: one growing byte buffer per device (PyTorch owns the memory).
# ------------------------------------------------------------------------------------------
_workspaces = {}


def workspace(device, nbytes):
    key = torch.device(device).index
    buf = _workspaces.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = None
        _workspaces[key] = None
        buf = torch.empty(int(nbytes * 1.1) + 4096, dtype=torch.uint8, device=device)
        _workspaces[key] = buf
    return buf


# ------------------------------------------------------------------------------------------
# Struct builders
# ------------------------------------------------------------------------------------------
def make_mlp_struct(sd, d_in, d_latent, d_hidden, d_out, n_blocks, combine_layer, packed=None):
    """sd: dict name -> contiguous fp32 CUDA tensor with ResnetFC state_dict keys.  A key missing from sd leaves its
    pointer NULL (a frozen tensor of a gradient struct for the _sel backward entry points)."""
    m = PnrMlp()
    m.d_in, m.d_latent, m.d_hidden, m.d_out = d_in, d_latent, d_hidden, d_out
    m.n_blocks, m.combine_layer = n_blocks, combine_layer
    p = lambda k: dptr(sd.get(k), k)
    m.lin_in_w, m.lin_in_b = p("lin_in.weight"), p("lin_in.bias")
    m.lin_out_w, m.lin_out_b = p("lin_out.weight"), p("lin_out.bias")
    for i in range(n_blocks):
        m.fc0_w[i], m.fc0_b[i] = p(f"blocks.{i}.fc_0.weight"), p(f"blocks.{i}.fc_0.bias")
        m.fc1_w[i], m.fc1_b[i] = p(f"blocks.{i}.fc_1.weight"), p(f"blocks.{i}.fc_1.bias")
    for i in range(min(combine_layer, n_blocks)):
        m.lin_z_w[i], m.lin_z_b[i] = p(f"lin_z.{i}.weight"), p(f"lin_z.{i}.bias")
    if packed is not None:
        m.packed = C.c_void_p(packed.data_ptr())
        m.packed_bytes = packed.numel() * packed.element_size()
    return m


def make_scene_struct(latent_nhwc, poses, focal, c, SB, NS, image_w, image_h, scale_x, scale_y,
                      proj_coarse=None, proj_fine=None):
    s = PnrScene()
    V, Hl, Wl, Cc = latent_nhwc.shape
    assert V == SB * NS
    s.latent_nhwc, s.poses, s.focal, s.c = dptr(latent_nhwc), dptr(poses), dptr(focal), dptr(c)
    s.n_focal, s.n_c = focal.shape[0], c.shape[0]
    s.SB, s.NS, s.Hl, s.Wl, s.C = SB, NS, Hl, Wl, Cc
    s.image_w, s.image_h = float(image_w), float(image_h)
    s.scale_x, s.scale_y = float(scale_x), float(scale_y)
    s.proj_coarse = dptr(proj_coarse)
    s.proj_fine = dptr(proj_fine)
    return s


def camera_grad(net, needs, dev):
    """PnrCameraGrad over zeroed buffers shaped as net.poses / net.focal / net.c, for those `needs` (three bools) asks
    for -> (struct, or None when nothing is asked for; (d_poses, d_focal, d_c) with None for the rest)."""
    ts = tuple(torch.zeros(t.shape, dtype=torch.float32, device=dev) if need else None
               for t, need in zip((net.poses, net.focal, net.c), needs))
    if all(t is None for t in ts):
        return None, ts
    return PnrCameraGrad(*(dptr(t) for t in ts)), ts


def pack_latent(latent_nchw):
    V, Cc, Hl, Wl = latent_nchw.shape
    out = torch.empty(V, Hl, Wl, Cc, dtype=torch.float32, device=latent_nchw.device)
    with torch.cuda.device(latent_nchw.device):
        check(lib().pnr_pack_latent(dptr(latent_nchw, "latent"), dptr(out), V, Cc, Hl, Wl,
                                    stream_ptr(latent_nchw.device)))
    return out
