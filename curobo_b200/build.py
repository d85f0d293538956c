"""Build the native libraries in-tree (nvcc cross-compiles sm_90a without a GPU).

  curobo_b200/lib/libcurobo_b200.so   -- the product: sm_90a kernels + C ABI (include/curobo_b200.h)
  tests/hostmath/libcb200_hostmath.so -- TEST-ONLY host build of the scalar math (CPU unit tests)
  oracle/_ref/libcurobo_ref.so        -- TEST-ONLY: the reference's own CUDA kernels, compiled from
  oracle/_ref/libcurobo_ref_legacy.so    /root/reference where they lie (only when that tree exists)
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "curobo_b200", "csrc")
LIBDIR = os.path.join(ROOT, "curobo_b200", "lib")
PRODUCT_SO = os.path.join(LIBDIR, "libcurobo_b200.so")
HOSTMATH_SO = os.path.join(ROOT, "tests", "hostmath", "libcb200_hostmath.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libcurobo_ref.so")
REFERENCE = os.environ.get("CUROBO_REFERENCE", "/root/reference")

# same numeric flags as the reference's NVRTC/pybind builds
# (curobo/_src/curobolib/backends/cuda_core_backend/kernel_config.py:52-59)
NUMERIC = ["--ftz=true", "--fmad=true", "--prec-div=false", "--prec-sqrt=false"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _nvcc() -> str:
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _newer(target: str, sources) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("build failed: " + " ".join(cmd))
    if verbose and (r.stdout or r.stderr):
        print(r.stdout + r.stderr)


def _digest(paths) -> str:
    """Content hash of the sources: unlike mtimes it survives the copy onto the GPU box unchanged."""
    import hashlib
    h = hashlib.sha256()
    for p in paths:
        h.update(os.path.basename(p).encode())
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def build_product(force: bool = False, verbose: bool = False) -> str:
    """Up to date <=> the stamp next to the library holds the content hash of the sources (so an edited csrc/ never runs
    a stale binary, and a fresh copy of the tree with new mtimes does not rebuild)."""
    srcs = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))] + [os.path.join(ROOT, "include", "curobo_b200.h")]
    out, stamp = PRODUCT_SO, PRODUCT_SO + ".stamp"
    digest = _digest(srcs)

    def fresh() -> bool:
        if not os.path.exists(out) or not os.path.exists(stamp):
            return False
        with open(stamp) as f:
            return f.read().strip() == digest
    if not force and fresh():
        return out
    os.makedirs(LIBDIR, exist_ok=True)
    import fcntl
    lock = open(os.path.join(LIBDIR, ".build.lock"), "w")
    fcntl.flock(lock, fcntl.LOCK_EX)          # several ranks may start at once: one builds, the others wait and re-check
    try:
        if not force and fresh():
            return out
        return _build_product_locked(out, stamp, digest, verbose)
    finally:
        fcntl.flock(lock, fcntl.LOCK_UN)
        lock.close()


def _build_product_locked(out: str, stamp: str, digest: str, verbose: bool) -> str:
    cmd = [_nvcc(), "-std=c++17", "-O3", "-lineinfo", *ARCH, *NUMERIC, "-Xcompiler", "-fPIC", "-shared",
           "-Xptxas", "-v" if verbose else "-O3", "-o", out, "-lcudart"]
    # three translation units (rollout, trajectory and optimizer kernels), compiled concurrently then linked
    units = ["cb200_kernels.cu", "cb200_trajectory.cu", "cb200_optim.cu", "cb200_dynamics.cu", "cb200_edt.cu"]
    objs = [os.path.join(LIBDIR, u[:-3] + ".o") for u in units]
    flags = [c for c in cmd[1:] if c not in ("-shared", "-o", out, "-lcudart")]
    procs = [subprocess.Popen([cmd[0], *flags, "-c", os.path.join(CSRC, u), "-o", o], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for u, o in zip(units, objs)]
    logs = [p.communicate()[0] for p in procs]
    if verbose:
        print("\n".join(logs))
    if any(p.returncode != 0 for p in procs):
        sys.stderr.write("\n".join(logs))
        raise RuntimeError("build failed: nvcc -c " + " ".join(units))
    tmp = out + ".tmp"
    _run([cmd[0], *ARCH, "-shared", "-Xcompiler", "-fPIC", *objs, "-o", tmp, "-lcudart"], verbose)
    os.replace(tmp, out)
    with open(stamp, "w") as f:
        f.write(digest)
    for o in objs:
        os.remove(o)
    return out


def build_hostmath(force: bool = False, verbose: bool = False) -> str:
    src = os.path.join(ROOT, "tests", "hostmath", "cb200_hostmath.cu")
    deps = [src, os.path.join(CSRC, "cb200_math.cuh"), os.path.join(CSRC, "cb200_bspline.cuh"),
            os.path.join(CSRC, "cb200_dynamics.cuh"), os.path.join(CSRC, "cb200_edt.cuh")]
    if not force and _newer(HOSTMATH_SO, deps):
        return HOSTMATH_SO
    cmd = [_nvcc(), "-std=c++17", "-O2", *ARCH, *NUMERIC, "-Xcompiler", "-fPIC", "-shared", src, "-o", HOSTMATH_SO,
           "-lcudart"]
    _run(cmd, verbose)
    return HOSTMATH_SO


def build_reference_kernels(force: bool = False, verbose: bool = False):
    """oracle/_ref: the reference's CUDA kernels for FK fwd / FK bwd / self-collision, compiled from the
    reference tree (headers are included by path; nothing is copied).  Returns None if the tree is absent."""
    src = os.path.join(ROOT, "oracle", "ref_kernels_launcher.cu")
    kdir = os.path.join(REFERENCE, "curobo", "_src", "curobolib", "kernels")
    if not os.path.isdir(kdir) or not os.path.exists(src):
        return REF_SO if os.path.exists(REF_SO) else None
    if not force and _newer(REF_SO, [src]):
        return REF_SO
    os.makedirs(os.path.dirname(REF_SO), exist_ok=True)
    cmd = [_nvcc(), "-std=c++17", "-O3", "-lineinfo", *ARCH, *NUMERIC, "-Xcompiler", "-fPIC", "-shared",
           "-I", kdir, "-I", os.path.join(kdir, "common"), "-I", os.path.join(kdir, "third_party"),
           "-I", os.path.join(kdir, "kinematics"), "-I", os.path.join(kdir, "geometry", "self_collision"),
           "-I", os.path.join(kdir, "trajectory"), "-I", os.path.join(kdir, "trajectory", "bspline"),
           "-I", os.path.join(kdir, "optimization", "lbfgs"), "-I", os.path.join(kdir, "optimization", "line_search"),
           "-I", os.path.join(kdir, "dynamics"), "-I", os.path.join(kdir, "parallel_banding"),
           src, "-o", REF_SO, "-lcudart"]
    _run(cmd, verbose)
    return REF_SO


def build_reference_legacy_kernels(force: bool = False, verbose: bool = False):
    """oracle/_ref/libcurobo_ref_legacy.so: the reference's legacy trajectory kernels (POSITION clique, ACCELERATION
    integration), compiled from the reference tree like build_reference_kernels.  Returns None if the tree is absent."""
    src = os.path.join(ROOT, "oracle", "ref_legacy_trajectory_launcher.cu")
    out = os.path.join(os.path.dirname(REF_SO), "libcurobo_ref_legacy.so")
    kdir = os.path.join(REFERENCE, "curobo", "_src", "curobolib", "kernels")
    if not os.path.isdir(kdir) or not os.path.exists(src):
        return out if os.path.exists(out) else None
    if not force and _newer(out, [src]):
        return out
    os.makedirs(os.path.dirname(out), exist_ok=True)
    _run([_nvcc(), "-std=c++17", "-O3", "-lineinfo", *ARCH, *NUMERIC, "-Xcompiler", "-fPIC", "-shared", "-I", kdir, src, "-o",
          out, "-lcudart"], verbose)
    return out


def build_reference_callsites(force: bool = False, verbose: bool = False):
    """oracle/_ref/pyref: the reference's Python call sites of the kernel backends (cuda_ops/*.py and their import closure)
    compiled to byte code from the sources where they lie (recipe: oracle/build_pyref.py, run through
    oracle/build_pyref_particle.py, which adds the reference's MPPI optimizer; test infrastructure, git-ignored, travels to the
    GPU box).  Returns the directory, or None when /root/reference is absent and nothing was built before."""
    out = os.path.join(ROOT, "oracle", "_ref", "pyref")
    manifest = os.path.join(out, "MANIFEST.json")
    recipes = [os.path.join(ROOT, "oracle", f) for f in ("build_pyref.py", "build_pyref_particle.py")]
    recipe = recipes[-1]
    if not os.path.isdir(REFERENCE) or not all(os.path.exists(r) for r in recipes):
        return out if os.path.exists(manifest) else None
    if not force and _newer(manifest, recipes):
        return out
    _run([sys.executable, recipe], verbose)          # own process: the recipe installs import stubs
    return out


def build_all(force: bool = False, verbose: bool = False):
    build_reference_callsites(force, verbose)
    build_reference_legacy_kernels(force, verbose)
    return build_product(force, verbose), build_hostmath(force, verbose), build_reference_kernels(force, verbose)


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv, verbose=True))
