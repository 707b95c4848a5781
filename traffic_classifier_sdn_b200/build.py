"""Build libtcsdn.so in-tree with nvcc for sm_90a (H100).  No JIT cache, no torch extension machinery:
the .so sits next to the sources so that it travels to the GPU box with the repository snapshot."""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libtcsdn.so")
SOURCES = ["abi.cu", "scorers.cu", "forest.cu", "knn.cu", "svc.cu", "flow.cu", "knn_engine.cu", "svc_engine.cu", "comm.cu", "fit.cu"]
# scorers.cu is compiled five times: once as the dispatcher and once per tiled feature count (object name -> extra flags)
VARIANTS = {"scorers.cu": [("scorers.o", []), ("scorers_d4.o", ["-DTCSDN_SCORER_D=4"]), ("scorers_d8.o", ["-DTCSDN_SCORER_D=8"]),
                           ("scorers_d12.o", ["-DTCSDN_SCORER_D=12"]), ("scorers_d16.o", ["-DTCSDN_SCORER_D=16"])]}
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "tcsdn.h")]
    return any(os.path.getmtime(p) > t for p in deps)


def build(force=False, verbose=False):
    """Compile every .cu for sm_90a and link libtcsdn.so.  Returns the library path."""
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    env = dict(os.environ)
    env.pop("CC", None)
    env.pop("CXX", None)
    procs = []
    for src in SOURCES:
        for objname, vflags in VARIANTS.get(src, [(src.replace(".cu", ".o"), [])]):
            obj = os.path.join(objdir, objname)
            cmd = [nvcc, "-ccbin", "/usr/bin/g++"] + NVCC_FLAGS + vflags + ["-c", os.path.join(CSRC, src), "-o", obj]
            procs.append((f"{src} {' '.join(vflags)}".strip(), obj,
                          subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, env=env, text=True)))
    objs, log = [], []
    for src, obj, p in procs:
        out = p.communicate()[0]
        log.append(f"==== {src}\n{out}")
        if p.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {src}")
        objs.append(obj)
    with open(os.path.join(objdir, "ptxas.log"), "w") as fh:
        fh.write("\n".join(log))
    cmd = [nvcc, "-ccbin", "/usr/bin/g++", "-shared"] + NVCC_FLAGS[:2] + ["-o", LIB] + objs + ["-lcuda", "-ldl"]
    subprocess.check_call(cmd, env=env)
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
