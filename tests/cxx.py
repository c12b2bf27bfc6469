"""Compiling and running the C++ and CUDA test programs: syntax checks of the drop-in headers, programs linked against
libcilantro_b200, host builds of the rule headers and the nvcc / g++ builds of the device harnesses.

    import cxx
    exe = cxx.build(os.path.join(ROOT, "examples", "segment_cloud.cpp"), str(tmp_path / "segment_cloud"))
    out = cxx.run(exe, cwd=str(tmp_path))
"""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INC = os.path.join(ROOT, "include")
CSRC = os.path.join(ROOT, "cilantro_b200", "csrc")
LIBDIR = os.path.join(ROOT, "cilantro_b200")
EIGEN_STUB = os.path.join(ROOT, "tests", "cpp", "eigen_stub")


def env():
    """The environment without CXX / CC (a compiler wrapper may be exported there): the programs use the PATH g++."""
    e = dict(os.environ)
    e.pop("CXX", None)
    e.pop("CC", None)
    return e


def syntax(path=None, src=None, flags=("-Wall",)):
    """g++ -fsyntax-only of the file `path` or of the source text `src` against include/: the completed process, so
    that a negative test can assert on its stderr."""
    cmd = ["g++", "-std=c++17", "-fsyntax-only", "-I", INC, *flags]
    if src is None:
        return subprocess.run(cmd + [path], capture_output=True, text=True, env=env())
    return subprocess.run(cmd + ["-x", "c++", "-"], input=src, capture_output=True, text=True, env=env())


def build(src, exe, flags=("-O2",), link=True):
    """g++ src -o exe with `flags`; link: against include/ and libcilantro_b200 (library directory and rpath)."""
    cmd = ["g++", "-std=c++17"] + (["-I", INC] if link else []) + [*flags, src, "-o", exe]
    if link:
        cmd += ["-L", LIBDIR, "-lcilantro_b200", f"-Wl,-rpath,{LIBDIR}"]
    subprocess.check_call(cmd, env=env())
    return exe


def run(exe, *args, timeout=300, cwd=None):
    """Runs a test program, asserts a zero exit code and returns its stdout (also printed)."""
    out = subprocess.run([exe, *map(str, args)], capture_output=True, text=True, timeout=timeout, cwd=cwd)
    print(out.stdout)
    assert out.returncode == 0, out.stdout + out.stderr
    return out.stdout


def eigen_flags():
    """[] where a real Eigen is installed, else the include flags of the stand-in tests/cpp/eigen_stub."""
    real = subprocess.run(["g++", "-std=c++17", "-E", "-x", "c++", "-"], input="#include <Eigen/Dense>\n", text=True,
                          capture_output=True, env=env()).returncode == 0
    return [] if real else ["-I", EIGEN_STUB]


def harness(src, exe, inc, device):
    """A device harness of tests/cuda: nvcc with the library's own flags (cilantro_b200/build.py NVCC_FLAGS) when
    `device`, else g++ on the same source as C++. inc: the -I flags."""
    if device:
        from cilantro_b200 import build as cb_build

        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        cmd = [nvcc] + cb_build.NVCC_FLAGS + ["-ccbin", "g++"] + list(inc) + ["-o", exe, src]
    else:
        cmd = ["g++", "-x", "c++", "-std=c++17", "-O2"] + list(inc) + ["-o", exe, src]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env())
    assert r.returncode == 0, r.stdout + r.stderr
    return exe
