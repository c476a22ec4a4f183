"""Build an alternative libdfx.so with extra -D flags for same-box A/B timing (dev tool):
    python tools/build_ab.py <tag> [-DFLAG=VALUE ...]      ->  build/ablib/libdfx_<tag>.so   (load it with DFX_LIBRARY=...)"""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g

tag, extra = sys.argv[1], sys.argv[2:]
objdir = os.path.join(ROOT, "build", "ab", "obj_" + tag)
os.makedirs(objdir, exist_ok=True)
nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
procs, objs = [], []
for name, src, flags in g.UNITS:
    obj = os.path.join(objdir, name + ".o")
    objs.append(obj)
    procs.append(subprocess.Popen([nvcc] + g.NVCC_FLAGS + flags + extra + ["-c", "-o", obj, os.path.join(g.CSRC, src)], cwd=ROOT))
assert all(p.wait() == 0 for p in procs)
os.makedirs(os.path.join(ROOT, "build", "ablib"), exist_ok=True)
out = os.path.join(ROOT, "build", "ablib", "libdfx_%s.so" % tag)
subprocess.check_call([nvcc, "-arch=sm_90a", "-shared", "-o", out] + objs, cwd=ROOT)
print(out)
