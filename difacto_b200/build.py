"""Build the sm_90a (H100) engine in-tree: difacto_b200/lib/libdifacto_b200.so.

nvcc cross-compiles without a GPU.  The .so is a build product and is git-ignored.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libdifacto_b200.so")
SOURCES = ["kernels_fm.cu", "kernels_table.cu", "kernels_localize.cu", "kernels_shard.cu", "kernels_checkpoint.cu",
           "kernels_prune.cu", "engine.cu", "shard.cu", "checkpoint.cu", "growth.cu", "prune.cu"]
HEADERS = ["dfb_internal.cuh", "dfb_device.cuh", "engine_internal.cuh", "shard_layout.cuh",
           os.path.join("..", "..", "include", "difacto_b200.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC,-O2,-Wall", "--expt-relaxed-constexpr", "-Xptxas", "-v",
         "-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"]
FLAGS += os.environ.get("DFB_EXTRA_NVCC_FLAGS", "").split()      # tuning experiments (e.g. -DDFB_FM_MINBLOCKS=4)


def _digest():
    h = hashlib.sha256()
    for f in SOURCES + HEADERS:
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.stamp")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(LIBDIR, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [NVCC] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out = p.communicate()[0]
        log.append(f"==== {src} ====\n{out}")
        if p.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {src}")
    with open(os.path.join(LIBDIR, "ptxas.log"), "w") as fh:
        fh.write("\n".join(log))
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-cudart", "static", "-ccbin",
                                                  "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"]
    subprocess.check_call(cmd)
    with open(stamp, "w") as fh:
        fh.write(dig)
    if verbose:
        print("\n".join(log))
    return LIB


def build_variant(name, extra_flags):
    """a tuning build with extra nvcc flags -> lib/variants/<name>.so (load it with DFB_LIB=...; never the product)"""
    vdir = os.path.join(LIBDIR, "variants", name)
    os.makedirs(vdir, exist_ok=True)
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(vdir, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [NVCC] + [f for f in FLAGS if f not in ("-Xptxas", "-v")] + list(extra_flags) + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out = p.communicate()[0]
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {src}")
    lib = os.path.join(LIBDIR, "variants", name + ".so")
    subprocess.check_call([NVCC, "-shared", "-o", lib] + objs + ["-cudart", "static", "-ccbin",
                                                                 "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"])
    for o in objs:
        os.remove(o)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
