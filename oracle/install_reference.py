"""Install the reference (NVlabs/DiffRL) into the git-ignored ``baseline/_ref/`` so that it TRAVELS to the GPU box.

TEST / BENCH INFRASTRUCTURE ONLY (build container: ``/root/reference`` does not exist on the GPU box).

    python oracle/install_reference.py [--no-cuda]

What lands in ``baseline/_ref/`` (never in git history; shipped by gpurun like the built ``.so`` files):

* ``refdflex/dflex/``   the reference's own ``dflex`` package (``dflex/dflex`` of the reference), with the
  NON-NUMERICAL edits listed in ``PATCHES`` below and nothing else;
* ``envs/ utils/ algorithms/ models/ examples/cfg/``   byte-for-byte copies;
* ``refdflex/dflex/kernels/``   the reference's generated C++/CUDA kernels, built HERE by the reference's own
  ``compile()`` (cross-compiled for sm_90; the reference ships ``compute_35`` PTX only, which nvcc 12.9 rejects).

Two things use it, both on the GPU box:

1. ``bench.py --impl reference-cuda`` -- the reference's own CUDA path driven through its stock ``envs`` (the
   "second bar" of SURVEY.md section 8d): ``sys.path = [oracle/refshim, baseline/_ref/refdflex, baseline/_ref]``;
2. ``tests/test_gpu_dropin.py`` -- the reference's UNCHANGED ``envs/*.py`` / ``algorithms/shac.py`` on top of THIS
   repo's ``dflex``: ``sys.path = [repo root, oracle/refshim, baseline/_ref]``.
"""
import argparse
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("DIFFRL_REFERENCE", "/root/reference")
DST = os.path.join(ROOT, "baseline", "_ref")

# (file, old, new, why) -- literal substring edits of the COPY; none touches the arithmetic of the hot path
PATCHES = [
    ("adjoint.py", "node.slice.value", "node.slice",
     "ast.Index no longer wraps subscripts (Python >= 3.9)"),
    ("adjoint.py", "-gencode=arch=compute_35,code=compute_35", "-gencode=arch=compute_90,code=sm_90",
     "adjoint.py:1861: nvcc 12.9 has no compute_35; build the generated kernels for the H100"),
    ("adjoint.py", "    use_cuda = torch.cuda.is_available()\n",
     "    use_cuda = torch.cuda.is_available() or os.environ.get('DFLEX_FORCE_CUDA_BUILD') == '1'\n",
     "adjoint.py:1750: allow cross-compiling the CUDA module in the GPU-less build container"),
    ("adjoint.py", "            if (torch.cuda.is_available()):\n                self.forward_cuda",
     "            if (torch.cuda.is_available() or os.environ.get('DFLEX_FORCE_CUDA_BUILD') == '1'):\n                self.forward_cuda",
     "adjoint.py:1737: same, for the entry-point lookup"),
]

COPY_DIRS = ["envs", "utils", "algorithms", "models"]


def _copy_tree(src, dst):
    if os.path.exists(dst):
        shutil.rmtree(dst)
    shutil.copytree(src, dst, ignore=shutil.ignore_patterns("__pycache__", "*.pyc", "kernels"))
    os.chmod(dst, 0o755)
    for base, dirs, files in os.walk(dst):       # the reference tree is read-only; the copy must not be
        for name in dirs:
            os.chmod(os.path.join(base, name), 0o755)
        for name in files:
            os.chmod(os.path.join(base, name), 0o644)


def install(with_cuda=True):
    if not os.path.isfile(os.path.join(REF, "dflex", "dflex", "sim.py")):
        raise SystemExit("reference tree not found at %s" % REF)
    os.makedirs(DST, exist_ok=True)
    pkg = os.path.join(DST, "refdflex", "dflex")
    keep = None
    kern = os.path.join(pkg, "kernels")
    if os.path.isdir(kern):                       # keep a finished build across re-installs (cache keyed on the source string)
        keep = os.path.join(DST, "_kernels_keep")
        if os.path.exists(keep):
            shutil.rmtree(keep)
        shutil.move(kern, keep)
    _copy_tree(os.path.join(REF, "dflex", "dflex"), pkg)
    if keep:
        shutil.move(keep, kern)
    for fname, old, new, _why in PATCHES:
        path = os.path.join(pkg, fname)
        text = open(path).read()
        if old not in text:
            raise SystemExit("patch target %r not found in %s" % (old, path))
        open(path, "w").write(text.replace(old, new))
    for d in COPY_DIRS:
        _copy_tree(os.path.join(REF, d), os.path.join(DST, d))
    os.makedirs(os.path.join(DST, "examples"), exist_ok=True)
    _copy_tree(os.path.join(REF, "examples", "cfg"), os.path.join(DST, "examples", "cfg"))
    with open(os.path.join(DST, "README.txt"), "w") as f:
        f.write("Installed by oracle/install_reference.py from %s; git-ignored; edits to refdflex/dflex/adjoint.py:\n" % REF)
        for fname, old, new, why in PATCHES:
            f.write("  %s: %r -> %r  (%s)\n" % (fname, old, new, why))
    # build the generated kernels (CPU + CUDA) with the reference's own compile(), in a fresh interpreter
    env = dict(os.environ)
    env["DFLEX_FORCE_CUDA_BUILD"] = "1" if with_cuda else "0"
    env.setdefault("CUDA_HOME", "/usr/local/cuda")
    env["TORCH_CUDA_ARCH_LIST"] = "9.0"
    env.setdefault("MAX_JOBS", "8")
    code = ("import sys, numpy as np; np.Inf = np.inf; sys.path[:0] = [%r, %r, %r]; import dflex; print('reference dflex built:', dflex.__file__)"
            % (os.path.join(HERE, "refshim"), os.path.join(DST, "refdflex"), DST))
    subprocess.check_call([sys.executable, "-c", code], env=env, cwd=DST)
    print("installed reference into", DST)


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-cuda", action="store_true")
    a = ap.parse_args()
    install(with_cuda=not a.no_cuda)
