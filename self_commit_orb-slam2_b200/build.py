"""Builds libb200slam.so (sm_90a only) in-tree with nvcc, and the CPU oracle with g++.

The .so files are build products and git-ignored.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200slam.so")
ORACLE_DIR = os.path.join(ROOT, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "liborb_oracle.so")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]  # H100 (Hopper)
NVCC_FLAGS = GENCODE + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC,-O3"]
# extractor/matcher/keyframe database: bit-exact float arithmetic, never contract a*b+c; LocalBA is FP64 with a 1e-5 bar
# -> FMA allowed; the essential graph differentiates numerically (delta = 1e-9 amplifies last-bit differences ~5e8 times)
NO_FMAD = {"extractor.cu", "extractor_tile.cu", "matcher.cu", "common.cu", "kfdb.cu", "essential.cu", "sim3opt.cu",
            "initializer.cu", "sim3solver.cu", "pnpsolver.cu"}


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def cuda_sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _deps_of(src):
    """Files whose change makes `src`'s object stale (the include graph of csrc/ is small and fixed); this file carries
    the architecture and compiler flags."""
    base = os.path.basename(src)
    deps = [src, os.path.join(CSRC, "common.cuh"), os.path.join(ROOT, "include", "b200slam.h"), os.path.abspath(__file__)]
    if base.startswith("extractor"):
        deps.append(os.path.join(CSRC, "extractor.cuh"))
    if base in ("localba.cu", "gba.cu", "essential.cu", "sim3opt.cu"):
        deps.append(os.path.join(CSRC, "ba_math.cuh"))
        deps.append(os.path.join(CSRC, "levenberg.cuh"))
    if base in ("essential.cu", "sim3opt.cu"):
        deps.append(os.path.join(CSRC, "sim3.cuh"))
    if base in ("gba.cu", "essential.cu"):
        deps.append(os.path.join(CSRC, "chol.cuh"))
    if base in ("initializer.cu", "pnpsolver.cu"):
        deps.append(os.path.join(CSRC, "jacobi.cuh"))
    if base == "extractor.cu":
        deps.append(os.path.join(ROOT, "data", "orb_pattern_31.inc"))
    return deps


def build_cuda(force=False, verbose=False):
    srcs = cuda_sources()
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    for s in srcs:
        o = s[:-3] + ".o"
        objs.append(o)
        if not force and not verbose and _newer(o, _deps_of(s)):
            continue  # object up to date (localba.cu alone takes minutes to compile)
        cmd = [nvcc] + NVCC_FLAGS + (["--fmad=false"] if os.path.basename(s) in NO_FMAD else []) + (
            ["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out.decode())
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    if not procs and not force and _newer(LIB, objs):
        return LIB
    cmd = [nvcc, "-shared"] + GENCODE + ["-o", LIB] + objs + ["-lcudart"]
    subprocess.check_call(cmd)
    return LIB


def build_oracle(force=False):
    srcs = [os.path.join(ORACLE_DIR, f) for f in os.listdir(ORACLE_DIR) if f.endswith((".cpp", ".h"))]
    srcs.append(os.path.join(ROOT, "data", "orb_pattern_31.inc"))
    if force or not _newer(ORACLE_LIB, srcs):
        subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-B", "liborb_oracle.so"])
    # the keyframe database's CPU restatement (oracle/kfdb.mk)
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "kfdb.mk"] + (["-B"] if force else []) + ["liborb_kfdb.so"])
    # the global bundle adjustment's CPU restatement (oracle/gba.mk)
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "gba.mk"] + (["-B"] if force else []) + ["liborb_gba.so"])
    # the essential graph's CPU restatement (oracle/essential.mk)
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "essential.mk"] + (["-B"] if force else []) +
                          ["liborb_essential.so"])
    # OptimizeSim3's CPU restatement (oracle/sim3opt.mk)
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "sim3opt.mk"] + (["-B"] if force else []) +
                          ["liborb_sim3opt.so"])
    # the monocular initialiser's CPU restatement (oracle/init.mk)
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "init.mk"] + (["-B"] if force else []) +
                          ["liborb_init.so"])
    # the Sim3 RANSAC's CPU restatement (oracle/sim3solver.mk)
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "sim3solver.mk"] + (["-B"] if force else []) +
                          ["liborb_sim3solver.so"])
    # the EPnP RANSAC's CPU restatement (oracle/pnpsolver.mk)
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "-f", "pnpsolver.mk"] + (["-B"] if force else []) +
                          ["liborb_pnpsolver.so"])
    return ORACLE_LIB


def build_oracle_ref():
    """oracle/_ref: the reference's own sources compiled in place against oracle/refshim (only where the reference's
    sources are present, at B2S_REFERENCE_ROOT; elsewhere prebuilt files are used).  Checker infrastructure, never
    product."""
    ref = os.environ.get("B2S_REFERENCE_ROOT", "/root/reference")
    if not os.path.isdir(os.path.join(ref, "src")):
        return None
    subprocess.check_call(["make", "-s", "-j8", "-C", ORACLE_DIR, "ref", "REF=" + ref])
    subprocess.check_call(["make", "-s", "-j8", "-C", ORACLE_DIR, "-f", "kfdb.mk", "ref", "REF=" + ref])
    subprocess.check_call(["make", "-s", "-j8", "-C", ORACLE_DIR, "-f", "gba.mk", "gba-ref", "REF=" + ref])
    subprocess.check_call(["make", "-s", "-j8", "-C", ORACLE_DIR, "-f", "essential.mk", "essential-ref", "REF=" + ref])
    subprocess.check_call(["make", "-s", "-j8", "-C", ORACLE_DIR, "-f", "sim3opt.mk", "sim3opt-ref", "REF=" + ref])
    subprocess.check_call(["make", "-s", "-j8", "-C", ORACLE_DIR, "-f", "init.mk", "init-ref", "REF=" + ref])
    subprocess.check_call(["make", "-s", "-j8", "-C", ORACLE_DIR, "-f", "sim3solver.mk", "sim3solver-ref", "REF=" + ref])
    subprocess.check_call(["make", "-s", "-j8", "-C", ORACLE_DIR, "-f", "pnpsolver.mk", "pnpsolver-ref", "REF=" + ref])
    return os.path.join(ORACLE_DIR, "_ref")


if __name__ == "__main__":
    build_cuda(force="--force" in sys.argv, verbose="-v" in sys.argv)
    build_oracle(force="--force" in sys.argv)
    build_oracle_ref()
    print("built", LIB, ORACLE_LIB)
