"""In-tree build of libvdo_b200.so (nvcc, sm_90a only).  Called by __graft_entry__.build().

Every source is compiled to its own object (in parallel, only when stale) and linked into one shared library.  Files
listed in PER_FILE get extra flags: pnp_ransac.cu is compiled with --fmad=false so that its double-precision minimal
solver rounds like the C oracle (gcc -ffp-contract=off) and hypotheses score identically on both sides; obj_motion.cu so
that its 4x4 products, inverse and back-projection round as the tracker's host helpers do; cam_motion.cu for the same reason."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
OUT = os.path.join(HERE, "libvdo_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
         "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
PER_FILE = {"pnp_ransac.cu": ["--fmad=false"], "obj_motion.cu": ["--fmad=false"], "cam_motion.cu": ["--fmad=false"]}


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))


def _compile(src: str, newest_header: float, force: bool):
    obj = os.path.join(OBJ, os.path.basename(src) + ".o")
    if not force and os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(src), newest_header):
        return obj, 0, ""
    cmd = [NVCC] + FLAGS + PER_FILE.get(os.path.basename(src), []) + ["-c", "-o", obj, src]
    r = subprocess.run(cmd, capture_output=True, text=True)
    return obj, r.returncode, " ".join(cmd) + "\n" + r.stdout + r.stderr


def build(force: bool = False, verbose: bool = False) -> str:
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))] + [os.path.join(HERE, "..", "include", "vdo_b200.h"), __file__]
    newest_header = max(os.path.getmtime(h) for h in headers)
    srcs = sources()
    if not force and os.path.exists(OUT) and all(os.path.getmtime(d) <= os.path.getmtime(OUT) for d in srcs + headers):
        return OUT
    os.makedirs(OBJ, exist_ok=True)
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(lambda s: _compile(s, newest_header, force), srcs))
    log = "".join(r[2] for r in res)
    bad = [r for r in res if r[1] != 0]
    rc = 1 if bad else 0
    if not bad:
        cmd = [NVCC] + ARCH + ["-shared", "-o", OUT] + [r[0] for r in res] + ["-lz"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log += " ".join(cmd) + "\n" + r.stdout + r.stderr
        rc = r.returncode
    with open(os.path.join(HERE, "build.log"), "a" if not force else "w") as f:
        f.write(log)
    if verbose or rc != 0:
        sys.stderr.write(log)
    if rc != 0:
        raise RuntimeError("nvcc failed building libvdo_b200.so (see vdo_slam_b200/build.log)")
    return OUT


if __name__ == "__main__":
    print(build(force=True, verbose="-v" in sys.argv))
