#!/usr/bin/env python
"""Install the UNMODIFIED reference (sxyu/pixel-nerf) inside the tree, and build the "overlay" tree that lets the
reference's own scripts run against this package.

  python oracle/install_ref.py                 # $PIXELNERF_REF (or /root/reference) -> oracle/_ref/ (build() does this)
  python oracle/install_ref.py --overlay DIR   # DIR/{eval,train,conf,expconf.conf} -> the reference's, DIR/src -> ours

`oracle/_ref/` is git-ignored (the reference is not product source and is never committed), but it is part of the
built tree, so a copy of the built tree carries it to the machine that runs the GPU tests.  There it is (a) the timing arm
`bench.py --impl reference` / `--impl reference-gpu` (the reference's own code, through its own public API) and
(b) the pass-through target of `_pnr_refpath` for everything outside the hot path (`data`, `model.loss`, ...).

The reference is pure Python (no setup.py / pyproject), so "install" = copy the five trees its scripts use.  Only
files are copied; nothing is edited.

Overlay: the reference's scripts start with `sys.path.insert(0, <dir of script>/../src)` (eval/gen_video.py:4-6,
train/train.py:7-9), which defeats PYTHONPATH.  The one supported drop-in install is therefore a directory that looks
like the reference checkout but whose `src/` is this package's `pixel-nerf_b200/src` -- symlinks only:

    DIR/eval, DIR/train, DIR/conf*, DIR/expconf.conf*  ->  the reference's      (* conf from this package when
    DIR/src                                            ->  pixel-nerf_b200/src     --our-conf is given)

and `python DIR/eval/gen_video.py ...` / `python DIR/train/train.py ...` run the UNMODIFIED scripts on the fused path.
"""
import argparse
import os
import shutil
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TREES = ["src", "conf", "eval", "train", "expconf.conf"]


INSTALLED = os.path.join(REPO, "oracle", "_ref")
CHECKOUTS = ("/root/reference",)   # conventional checkout location, after $PIXELNERF_REF


def find_source():
    """A reference checkout outside the repository: $PIXELNERF_REF, else the conventional location; None if absent
    or unreadable."""
    for root in (os.environ.get("PIXELNERF_REF"), *CHECKOUTS):
        if root and os.path.isdir(os.path.join(root, "src", "render")) and os.access(os.path.join(root, "src"), os.R_OK):
            return root
    return None


def find_reference():
    """The reference for tests and tools: $PIXELNERF_REF, else the copy build() installs at oracle/_ref, else the
    conventional checkout location."""
    for root in (os.environ.get("PIXELNERF_REF"), INSTALLED, *CHECKOUTS):
        if root and os.path.isdir(os.path.join(root, "src", "render")) and os.access(os.path.join(root, "src"), os.R_OK):
            return root
    return None


def install(dest=INSTALLED):
    """Copies the unmodified reference trees to `dest` (git-ignored); returns dest, or None without a checkout."""
    src_root = find_source()
    if src_root is None:
        return None
    if os.path.realpath(src_root) == os.path.realpath(dest):
        return dest
    os.makedirs(dest, exist_ok=True)
    for name in TREES:
        s, d = os.path.join(src_root, name), os.path.join(dest, name)
        if os.path.isdir(s):
            if os.path.exists(d):
                shutil.rmtree(d)
            shutil.copytree(s, d, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
        else:
            shutil.copy2(s, d)
    print(f"installed {src_root} -> {dest}")
    return dest


def make_overlay(dest, ref_root=None, our_conf=False):
    """Symlink tree described in the module docstring; returns dest."""
    ref_root = ref_root or find_reference()
    if ref_root is None:
        raise RuntimeError("no reference checkout found (set PIXELNERF_REF or run oracle/install_ref.py)")
    os.makedirs(dest, exist_ok=True)
    pkg = os.path.join(REPO, "pixel-nerf_b200")
    links = {"src": os.path.join(pkg, "src"), "eval": os.path.join(ref_root, "eval"),
             "train": os.path.join(ref_root, "train"),
             "conf": os.path.join(pkg if our_conf else ref_root, "conf"),
             "expconf.conf": os.path.join(pkg if our_conf else ref_root, "expconf.conf")}
    for name, target in links.items():
        p = os.path.join(dest, name)
        if os.path.islink(p):
            os.unlink(p)
        elif os.path.exists(p):
            raise RuntimeError(f"{p} exists and is not a symlink")
        os.symlink(os.path.abspath(target), p)
    return dest


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--dest", default=INSTALLED)
    ap.add_argument("--overlay", default=None, help="also (or only, if the reference is installed) build an overlay tree")
    ap.add_argument("--our-conf", action="store_true", help="overlay uses this package's conf/ instead of the reference's")
    a = ap.parse_args()
    if a.overlay is None:
        if install(a.dest) is None:
            raise SystemExit("no reference checkout found (set PIXELNERF_REF)")
    else:
        if find_reference() is None:
            raise SystemExit("no reference checkout found")
        print("overlay at", make_overlay(a.overlay, our_conf=a.our_conf))
    sys.exit(0)
