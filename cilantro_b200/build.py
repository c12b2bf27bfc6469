"""Build libcilantro_b200.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc.

nvcc cross-compiles without a GPU; the .so is a build product (git-ignored). `python -m cilantro_b200.build [--force] [-v] [-DNAME=VALUE ...] [--out=x.so]`.

Every translation unit is compiled to its own object under cilantro_b200/build/ (in parallel, re-done only
when the source, any header or the flags changed) and the objects are linked into the shared library.
"""
import concurrent.futures
import glob
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libcilantro_b200.so")
OBJ = os.path.join(HERE, "build")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-O2",
]
LINK_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-cudart", "static", "-Xcompiler", "-fPIC"]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cpp")))


def headers():
    return sorted(glob.glob(os.path.join(CSRC, "*.h*")) + glob.glob(os.path.join(CSRC, "*.cuh")) +
                  [os.path.join(HERE, "..", "include", "cilantro_b200.h"), __file__])


def _env():
    env = dict(os.environ)
    env.pop("CXX", None)  # the image exports a wrapper g++ without OpenMP specs; use the PATH compiler
    env.pop("CC", None)
    return env


def build(force=False, verbose=False, defines=(), out=None):
    """defines/out: build an experimental variant (e.g. defines=["CB_SEGMENT_COUNTERS=1"], out="libcilantro_b200_counters.so")."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    target = LIB if out is None else os.path.join(HERE, out)
    flags = NVCC_FLAGS + [f"-D{d}" for d in defines] + (["-Xptxas", "-v"] if verbose else [])
    tag = hashlib.sha1(" ".join(flags).encode()).hexdigest()[:10]
    objdir = os.path.join(OBJ, tag)
    os.makedirs(objdir, exist_ok=True)
    hdr_time = max(os.path.getmtime(h) for h in headers())
    jobs = []
    objs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        objs.append(obj)
        if force or verbose or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr_time):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [nvcc] + flags + ["-ccbin", "g++", "-c", "-o", obj, src]
        r = subprocess.run(cmd, env=_env(), capture_output=True, text=True)
        return src, r.returncode, r.stdout + r.stderr

    failed = []
    if jobs:
        with concurrent.futures.ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            for src, rc, log in ex.map(compile_one, jobs):
                if rc != 0 or verbose:
                    sys.stderr.write(f"---- {os.path.basename(src)} ----\n{log}\n")
                if rc != 0:
                    failed.append(src)
    if failed:
        raise RuntimeError("nvcc failed for: " + ", ".join(os.path.basename(f) for f in failed))
    if jobs or not os.path.exists(target) or any(os.path.getmtime(o) > os.path.getmtime(target) for o in objs):
        subprocess.check_call([nvcc] + LINK_FLAGS + ["-ccbin", "g++", "-o", target] + objs + ["-ldl"], env=_env())
    if out is not None or defines or verbose:  # experimental variants do not keep their objects around
        import shutil

        shutil.rmtree(objdir, ignore_errors=True)
    return target


if __name__ == "__main__":
    defs = [a[2:] for a in sys.argv[1:] if a.startswith("-D")]
    outs = [a[6:] for a in sys.argv[1:] if a.startswith("--out=")]
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, defines=defs, out=outs[0] if outs else None))
