"""Kernel-by-kernel SASS comparison of two builds of the library's translation units.

    python tools/sass_functions.py OLD_OBJ_DIR NEW_OBJ_DIR [--skip-envp] [--objects GLOB | --all]

Splits `cuobjdump -sass` of every object matching GLOB (default step_f*.o, the step translation units; host.o is the host unit with the
snapshot, RNG-identity, parameter-block, clock, peer and accessor kernels; jac_f*.o, grad_f*.o and psens_f*.o are the tangent-rollout
units; --all: every object of the build) by function (instruction addresses and the source-path
identifier removed) and compares each kernel with the one of the same name in the other build.  --skip-envp leaves out the ENVP instantiations (per-env parameter blocks: the
8th template argument of step_kernel / rollout_kernel), reset_kernel and the parameter draw they call, whose code a change to the per-env parameter path is expected to
touch; every other kernel must then be identical.  Prints one line per differing or missing kernel and a summary; exit code 1 if any
compared kernel differs.  No GPU needed.
"""
import glob
import hashlib
import os
import re
import subprocess
import sys


def functions(obj):
    out = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, name, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                funcs[name] = hashlib.sha1("\n".join(body).encode()).hexdigest()
            name, body = m.group(1), []
            continue
        if name is None or line.strip().startswith("identifier") or ".section" in line:
            continue
        body.append(" ".join(re.sub(r"/\*[0-9a-f]{4,}\*/", "", line).split()))  # the address column width varies with the object size
    if name:
        funcs[name] = hashlib.sha1("\n".join(body).encode()).hexdigest()
    return funcs


def demangle(names):
    out = subprocess.run(["cu++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.splitlines()
    return dict(zip(names, out))


def is_envp_or_reset(pretty):
    if "reset_kernel" in pretty or "redraw_env_params" in pretty:
        return True
    m = re.search(r"(step_kernel|rollout_kernel)<([^>]*)>", pretty)
    if not m:
        return False
    args = [a.strip() for a in m.group(2).split(",")]
    return len(args) >= 8 and args[7] in ("true", "(bool)1")


def main():
    old_dir, new_dir = sys.argv[1], sys.argv[2]
    skip = "--skip-envp" in sys.argv
    pattern = "*.o" if "--all" in sys.argv else (sys.argv[sys.argv.index("--objects") + 1] if "--objects" in sys.argv else "step_f*.o")
    same = differ = skipped = 0
    for new_obj in sorted(glob.glob(os.path.join(new_dir, pattern))):
        old_obj = os.path.join(old_dir, os.path.basename(new_obj))
        a, b = functions(old_obj), functions(new_obj)
        pretty = demangle(sorted(set(a) | set(b)))
        for name in sorted(set(a) | set(b)):
            if skip and is_envp_or_reset(pretty[name]):
                skipped += 1
                continue
            if a.get(name) == b.get(name):
                same += 1
            else:
                differ += 1
                print(f"DIFFERENT {os.path.basename(new_obj)}: {pretty[name]}")
    print(f"kernels with identical SASS: {same}, different: {differ}, skipped (ENVP / reset): {skipped}")
    return 1 if differ else 0


if __name__ == "__main__":
    sys.exit(main())
