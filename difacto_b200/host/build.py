"""Build the host-side C++ mirror (CLI + test binary) against the in-tree engine library."""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
OUT = os.path.join(HERE, "bin")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
FLAGS = ["-std=c++14", "-O2", "-Wall", "-Wextra", "-I", os.path.join(HERE, "include")]
LIBDIR = os.path.join(PKG, "lib")
LINK = ["-L", LIBDIR, "-ldifacto_b200", f"-Wl,-rpath,{LIBDIR}", "-Wl,-rpath,$ORIGIN/../../lib"]
TARGETS = {
    "difacto_b200": ["src/main.cc", "src/sgd_learner.cc"],
    "host_tests": ["tests/host_tests.cc", "src/sgd_learner.cc"],
    "prune_settings_tests": ["tests/prune_settings_tests.cc", "src/sgd_learner.cc"],
    "prune_rare_settings_tests": ["tests/prune_rare_settings_tests.cc", "src/sgd_learner.cc"],
    "batch_dump": ["tests/batch_dump.cc"],
}


def build(force=False):
    os.makedirs(OUT, exist_ok=True)
    h = hashlib.sha256()
    for root, _, files in os.walk(HERE):
        if root.startswith(OUT):
            continue
        for f in sorted(files):
            if f.endswith((".h", ".cc")):
                h.update(open(os.path.join(root, f), "rb").read())
    dig = h.hexdigest()
    stamp = os.path.join(OUT, "build.stamp")
    if not force and os.path.exists(stamp) and open(stamp).read() == dig and all(
            os.path.exists(os.path.join(OUT, t)) for t in TARGETS):
        return OUT
    for name, srcs in TARGETS.items():
        cmd = [CXX] + FLAGS + [os.path.join(HERE, s) for s in srcs] + ["-o", os.path.join(OUT, name)] + LINK
        subprocess.check_call(cmd)
    open(stamp, "w").write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
