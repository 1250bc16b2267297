"""Build libgemb200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m gym_electric_motor_b200.build [--force] [--verbose]

The step kernel's 200 instantiations are spread over twelve translation units (motor family x real, csrc/gemb200_step_tu.cu)
that compile in parallel, the rollout-Jacobian kernels over twelve more (csrc/gemb200_jac_tu.cu), the return-gradient kernels over another twelve
(csrc/gemb200_grad_tu.cu) and the parameter-sensitivity kernels over twelve more (csrc/gemb200_psens_tu.cu); objects go to build/ (git-ignored),
only the linked .so stays in the package.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
HEADERS = [os.path.join(CSRC, "gemb200_kernels.cuh"), os.path.join(CSRC, "gemb200_params.h"), os.path.join(CSRC, "gemb200_launch.cuh"),
           os.path.join(CSRC, "gemb200_model.h"), os.path.join(CSRC, "gemb200_jac.h"), os.path.join(CSRC, "gemb200_tangent.cuh"),
           os.path.join(HERE, "..", "include", "gemb200.h")]
SOURCES = [os.path.join(CSRC, "gemb200.cu"), os.path.join(CSRC, "gemb200_step_tu.cu"), os.path.join(CSRC, "gemb200_jac_tu.cu"),
           os.path.join(CSRC, "gemb200_grad_tu.cu"), os.path.join(CSRC, "gemb200_psens_tu.cu")]
OUT = os.path.join(HERE, "libgemb200.so")
OBJ_DIR = os.path.join(HERE, "..", "build", "gemb200")
# -fmad=false: no implicit contraction of a*b+c — every fused multiply-add of the kernels is written out (fm() in gemb200_kernels.cuh), so
# that all instantiations of the step (step / rollout kernel, AoS / SoA, PLAIN / general) round identically: bit-identical results
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]  # H100 (Hopper); the only target the library is built and tested for
NVCC_FLAGS = ARCH + ["-O3", "-std=c++17", "-fmad=false", "-Xcompiler", "-fPIC"]
# -lineinfo (source-level profiles) on the host unit and the fp32 kernels — the ones that are profiled; the fp64 units go without it: line
# tables are ~60 % of a unit's size
LINEINFO = ["-lineinfo"]
FAMILIES = (0, 1, 2, 3, 4, 5)  # gemb200_params.h: MotorFamily
REALS = ("float", "double")


def nvcc_path():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def is_stale(out=OUT):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in HEADERS + SOURCES if os.path.exists(d))


def _units(only=None):
    units = [("host", SOURCES[0], LINEINFO)]
    for fam in FAMILIES:
        for real in REALS:
            if only and (fam, real) not in only:
                continue
            units.append((f"step_f{fam}_{real}", SOURCES[1], [f"-DGEMB200_TU_FAM={fam}", f"-DGEMB200_TU_REAL={real}"] + (LINEINFO if real == "float" else [])))
    if not only:  # the rollout-Jacobian kernels (gemb200_jac_tu.cu): one unit per family x real, like the step kernels
        for fam in FAMILIES:
            for real in REALS:
                units.append((f"jac_f{fam}_{real}", SOURCES[2], [f"-DGEMB200_JAC_FAM={fam}", f"-DGEMB200_JAC_REAL={real}"]))
        for fam in FAMILIES:  # the return-gradient kernels (gemb200_grad_tu.cu), likewise
            for real in REALS:
                units.append((f"grad_f{fam}_{real}", SOURCES[3], [f"-DGEMB200_JAC_FAM={fam}", f"-DGEMB200_JAC_REAL={real}"]))
        for fam in FAMILIES:  # the parameter-sensitivity kernels (gemb200_psens_tu.cu), likewise
            for real in REALS:
                units.append((f"psens_f{fam}_{real}", SOURCES[4], [f"-DGEMB200_JAC_FAM={fam}", f"-DGEMB200_JAC_REAL={real}"]))
    return units


def build(force=False, verbose=False, out=OUT, defines=(), only=None, jobs=None):
    """Compile and link.  `defines`/`only`/`out` are for experiment builds (tools/build_variants.py): extra -D flags, a subset of
    (family, real) units — pass -DGEMB200_ONLY_FAM=<family> with only={(family, "float")} so that the host code does not reference
    the missing units (otherwise the library fails to LOAD, on purpose: no silent holes) — and another output path."""
    if not force and not is_stale(out):
        return out
    tag = hashlib.sha1(("|".join(defines) + "|" + os.path.abspath(out)).encode()).hexdigest()[:10]
    obj_dir = os.path.join(OBJ_DIR, tag)
    os.makedirs(obj_dir, exist_ok=True)
    nvcc = nvcc_path()
    extra = list(defines) + (["-Xptxas", "-v"] if verbose else [])

    def compile_one(unit):
        name, src, flags = unit
        obj = os.path.join(obj_dir, name + ".o")
        cmd = [nvcc] + NVCC_FLAGS + extra + flags + ["-c", "-o", obj, src]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        return obj, res

    units = _units(only)
    with ThreadPoolExecutor(max_workers=jobs or min(len(units), os.cpu_count() or 4)) as ex:
        results = list(ex.map(compile_one, units))
    objs = []
    for obj, res in results:
        if verbose or res.returncode != 0:
            sys.stdout.write(res.stdout)
        if res.returncode != 0:
            raise RuntimeError("nvcc failed building libgemb200.so")
        objs.append(obj)
    link = [nvcc, "-shared"] + ARCH + ["-o", out] + objs
    res = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        sys.stdout.write(res.stdout)
        raise RuntimeError("link of libgemb200.so failed")
    return out


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(OUT)
