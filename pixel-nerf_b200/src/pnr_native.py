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
ENGINE_AUTO, ENGINE_SIMT, ENGINE_TC = 0, 1, 2
ENGINES = {"auto": ENGINE_AUTO, "simt": ENGINE_SIMT, "tc": ENGINE_TC}

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


class PnrShard(C.Structure):
    _fields_ = [("scene", C.POINTER(PnrScene)), ("mlp_coarse", C.POINTER(PnrMlp)), ("mlp_fine", C.POINTER(PnrMlp)),
                ("noise", C.POINTER(PnrNoise)), ("workspace", _fp), ("workspace_bytes", C.c_size_t),
                ("rays_stage", _fp), ("stage", PnrRenderOut), ("stream", _fp)]


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
        for name in ("pnr_mgpu_create", "pnr_mgpu_destroy", "pnr_mgpu_broadcast", "pnr_mgpu_render"):
            getattr(L, name).restype = C.c_int
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
    """sd: dict name -> contiguous fp32 CUDA tensor with ResnetFC state_dict keys."""
    m = PnrMlp()
    m.d_in, m.d_latent, m.d_hidden, m.d_out = d_in, d_latent, d_hidden, d_out
    m.n_blocks, m.combine_layer = n_blocks, combine_layer
    m.lin_in_w, m.lin_in_b = dptr(sd["lin_in.weight"]), dptr(sd["lin_in.bias"])
    m.lin_out_w, m.lin_out_b = dptr(sd["lin_out.weight"]), dptr(sd["lin_out.bias"])
    for i in range(n_blocks):
        m.fc0_w[i] = sd[f"blocks.{i}.fc_0.weight"].data_ptr()
        m.fc0_b[i] = sd[f"blocks.{i}.fc_0.bias"].data_ptr()
        m.fc1_w[i] = sd[f"blocks.{i}.fc_1.weight"].data_ptr()
        m.fc1_b[i] = sd[f"blocks.{i}.fc_1.bias"].data_ptr()
        dptr(sd[f"blocks.{i}.fc_0.weight"]), dptr(sd[f"blocks.{i}.fc_1.weight"])
    for i in range(min(combine_layer, n_blocks)):
        m.lin_z_w[i] = sd[f"lin_z.{i}.weight"].data_ptr()
        m.lin_z_b[i] = sd[f"lin_z.{i}.bias"].data_ptr()
        dptr(sd[f"lin_z.{i}.weight"])
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


def pack_latent(latent_nchw):
    V, Cc, Hl, Wl = latent_nchw.shape
    out = torch.empty(V, Hl, Wl, Cc, dtype=torch.float32, device=latent_nchw.device)
    with torch.cuda.device(latent_nchw.device):
        check(lib().pnr_pack_latent(dptr(latent_nchw, "latent"), dptr(out), V, Cc, Hl, Wl,
                                    stream_ptr(latent_nchw.device)))
    return out
