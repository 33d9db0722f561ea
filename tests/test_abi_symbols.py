"""The C-ABI library loads (no GPU needed) and exports every function include/pnr.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    text = open(os.path.join(ROOT, "include", "pnr.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(pnr_[a-z_0-9]+)\s*\(", text)))


def test_header_declares_the_documented_surface():
    names = declared_functions()
    for must in ("pnr_render", "pnr_field_eval", "pnr_sample_coarse", "pnr_composite", "pnr_sample_fine",
                 "pnr_pack_latent", "pnr_pack_mlp", "pnr_project_latent", "pnr_last_error", "pnr_abi_version",
                 "pnr_gen_rays", "pnr_frames_u8", "pnr_render_backward", "pnr_field_backward", "pnr_gemm_nt",
                 "pnr_mgpu_create", "pnr_mgpu_broadcast", "pnr_mgpu_render", "pnr_mgpu_destroy"):
        assert must in names


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as ge
    lib_path = os.path.join(ROOT, "pixel-nerf_b200", "lib", "libpnr_sm90.so")
    if not os.path.exists(lib_path):
        ge.build()
    lib = ctypes.CDLL(lib_path)
    for name in declared_functions():
        assert hasattr(lib, name), f"{name} declared in pnr.h but not exported"
    lib.pnr_abi_version.restype = ctypes.c_int
    assert lib.pnr_abi_version() == 2


def test_python_binding_matches_header_struct_sizes():
    """ctypes mirrors must have the C layout: compile a tiny sizeof probe with gcc."""
    import subprocess
    import sys
    import tempfile
    sys.path.insert(0, os.path.join(ROOT, "pixel-nerf_b200", "src"))
    import pnr_native as pn
    src = '#include <stdio.h>\n#include "pnr.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(PnrScene), sizeof(PnrMlp), sizeof(PnrRenderCfg), sizeof(PnrNoise), sizeof(PnrRenderOut), sizeof(PnrShard));return 0;}\n'
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "p.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "p")
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe], check=True)
        sizes = list(map(int, subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()))
    assert sizes == [ctypes.sizeof(pn.PnrScene), ctypes.sizeof(pn.PnrMlp), ctypes.sizeof(pn.PnrRenderCfg),
                     ctypes.sizeof(pn.PnrNoise), ctypes.sizeof(pn.PnrRenderOut), ctypes.sizeof(pn.PnrShard)]
