"""Builds libmzb200.so in-tree with nvcc for sm_90a (no torch involved)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmzb200.so")
SOURCES = ["abi.cu", "ktimer.cu", "fc_search.cu", "fc_infer.cu", "tree_kernels.cu", "tree_wide.cu", "pipeline.cu", "resnet.cu", "conv_tc.cu", "conv_x3.cu", "small_tower.cu", "small_search.cu", "selfplay.cu", "cnn_stem.cu", "conv_wide.cu", "conv_wide256.cu", "reanalyse.cu", "user_env.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-fmad=false", "-diag-suppress", "177",                     # tree arithmetic must never be contracted; FMAs are explicit fmaf()
    "-Xcompiler", "-fPIC", "-Xcompiler", "-O2", "--expt-relaxed-constexpr",
] + os.environ.get("MZ_NVCC_EXTRA", "").split()        # e.g. -DMZ_DUAL_ISSUER for the experiment in conv_tc.cu


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "mzb200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def write_prelude(out_dir):
    """The NVRTC prelude of user environments (csrc/user_env.cuh and the philox.cuh it includes) and their epilogue
    (csrc/user_env_expert.cuh) as C++ string literals, so the library carries the headers it compiles user sources
    against."""
    parts = []
    for name, var in (("philox.cuh", "kPhiloxCuh"), ("user_env.cuh", "kUserEnvCuh"),
                      ("user_env_expert.cuh", "kUserEnvExpertCuh")):
        text = open(os.path.join(CSRC, name)).read()
        assert ")MZPRELUDE\"" not in text
        parts.append(f'static const char {var}[] = R"MZPRELUDE({text})MZPRELUDE";\n')
    path = os.path.join(out_dir, "user_env_prelude.inc")
    if not os.path.exists(path) or open(path).read() != "".join(parts):
        with open(path, "w") as f:
            f.write("".join(parts))


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    write_prelude(os.path.join(HERE, "build"))
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-I", os.path.join(HERE, "build"), "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- nvcc {src}\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    subprocess.check_call([NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-ldl"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
