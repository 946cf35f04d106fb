"""Builds world_b200/lib/libworld_b200.so with nvcc for sm_90a (in-tree, no torch involved)."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "build")
SOURCES = ["wb_api.cu", "wb_host.cu", "wb_rng.cu", "wb_cheaptrick.cu", "wb_d4c.cu", "wb_stonemask.cu", "wb_synthesis.cu", "wb_codec.cu", "wb_fileio.cu", "wb_matlab.cu",
           "wb_f0common.cu", "wb_dio.cu", "wb_harvest.cu", "wb_multi.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# -fmad=false: values that feed int casts / comparisons must round like the reference's x86-64 -O1
# build (SURVEY.md App. B2); hot loops use explicit fma() where contraction is harmless.
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-fmad=false",
         "-Xcompiler", "-fPIC", "-Xptxas", "-v", "-I", os.path.join(HERE, "..", "include")]


def _newer(src, obj):
    if not os.path.exists(obj):
        return True
    t = os.path.getmtime(obj)
    deps = [src] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    deps.append(os.path.join(HERE, "..", "include", "world_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(verbose=False, force=False, defines=(), tag=""):
    """tag / defines: an A/B variant (lib/libworld_b200_<tag>.so built with -D<define>...), loaded through
    WORLD_B200_LIB; the product library is the untagged one."""
    objdir = OBJDIR + ("_" + tag if tag else "")
    os.makedirs(LIBDIR, exist_ok=True)
    os.makedirs(objdir, exist_ok=True)
    out = os.path.join(LIBDIR, "libworld_b200%s.so" % ("_" + tag if tag else ""))
    flags = FLAGS + ["-D" + d for d in defines]
    # objects compiled with other flags (another architecture, say) are stale whatever their mtime
    stamp = os.path.join(objdir, "flags.txt")
    if not os.path.exists(stamp) or open(stamp).read() != " ".join(flags):
        force = True
    jobs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(objdir, s.replace(".cu", ".o"))
        if force or _newer(src, obj):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        r = subprocess.run([NVCC] + flags + ["-c", src, "-o", obj], capture_output=True, text=True)
        log = r.stdout + r.stderr
        with open(obj + ".ptxas.log", "w") as f:
            f.write(log)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{log}")
        return log

    with ThreadPoolExecutor(max_workers=8) as ex:
        logs = list(ex.map(compile_one, jobs))
    if verbose:
        for l in logs:
            print(l)
    objs = [os.path.join(objdir, s.replace(".cu", ".o")) for s in SOURCES]
    if jobs or not os.path.exists(out):
        r = subprocess.run([NVCC, "-shared", "-o", out] + objs + ["-lcudart", "-ldl"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    with open(stamp, "w") as f:
        f.write(" ".join(flags))
    return out


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
