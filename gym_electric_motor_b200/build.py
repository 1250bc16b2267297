"""Build libgemb200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m gym_electric_motor_b200.build [--force] [--verbose]

The step kernel's 200 instantiations are spread over twelve translation units (motor family x real, csrc/gemb200_step_tu.cu)
that compile in parallel.  The tangent-rollout kernels (csrc/gemb200_tangent.cuh) come from one source, csrc/gemb200_tangent_tu.cu,
compiled once per kind x family x real (kind = the output struct: JacOut rollout Jacobians, GradOut return gradients, PsOut parameter
sensitivities), 36 more units; objects go to build/ (git-ignored), only the linked .so stays in the package.
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
SOURCES = [os.path.join(CSRC, "gemb200.cu"), os.path.join(CSRC, "gemb200_step_tu.cu"), os.path.join(CSRC, "gemb200_tangent_tu.cu")]
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
TANGENT_KINDS = (("jac", "JacOut"), ("grad", "GradOut"), ("psens", "PsOut"))  # object prefix, output struct (gemb200_jac.h)


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


def _units():
    units = [("host", SOURCES[0], LINEINFO)]
    for fam in FAMILIES:
        for real in REALS:
            units.append((f"step_f{fam}_{real}", SOURCES[1], [f"-DGEMB200_TU_FAM={fam}", f"-DGEMB200_TU_REAL={real}"] + (LINEINFO if real == "float" else [])))
    # the tangent-rollout kernels: one unit per kind x family x real, like the step kernels
    for prefix, out in TANGENT_KINDS:
        for fam in FAMILIES:
            for real in REALS:
                units.append((f"{prefix}_f{fam}_{real}", SOURCES[2], [f"-DGEMB200_TAN_OUT={out}", f"-DGEMB200_JAC_FAM={fam}", f"-DGEMB200_JAC_REAL={real}"]))
    return units


def build(force=False, verbose=False, out=OUT, jobs=None):
    """Compile and link into `out`.  Another output path gives a second library with its own object directory, e.g. the build of
    another commit to compare against (GEMB200_LIB selects the library that _cabi loads); `jobs` caps the parallel nvcc processes."""
    if not force and not is_stale(out):
        return out
    tag = hashlib.sha1(("|" + os.path.abspath(out)).encode()).hexdigest()[:10]
    obj_dir = os.path.join(OBJ_DIR, tag)
    os.makedirs(obj_dir, exist_ok=True)
    nvcc = nvcc_path()
    extra = ["-Xptxas", "-v"] if verbose else []

    def compile_one(unit):
        name, src, flags = unit
        obj = os.path.join(obj_dir, name + ".o")
        cmd = [nvcc] + NVCC_FLAGS + extra + flags + ["-c", "-o", obj, src]
        res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        return obj, res

    units = _units()
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
