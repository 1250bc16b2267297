#!/bin/bash
# Is the device code of HEAD the same as that of commit $1?  Builds every translation unit of that commit in a scratch worktree and compares
# `cuobjdump -sass` of every object with the current build (instruction addresses and the source-path identifier line removed): the host
# unit, the 12 step units and the 12 units of each tangent-rollout kind (jac, grad, psens).
#   bash tools/sass_identity.sh 503c048        (no GPU needed; a full build of both trees)
#   bash tools/sass_identity.sh 503c048 --per-function   kernel by kernel instead (tools/sass_functions.py --all), leaving out the ENVP
#        step / rollout instantiations and reset_kernel, which share the objects with every other kernel
set -eu
ref=${1:?commit}
wt=$(mktemp -d /tmp/gemb200_sass_XXXX)
git worktree add -q "$wt" "$ref"
trap 'git worktree remove --force "$wt"' EXIT
(cd "$wt" && python -c "import sys; sys.path.insert(0, '$wt'); from gym_electric_motor_b200 import build as b; b.build(force=True, out='$wt/lib_ref.so')" > /dev/null)
python -c "from gym_electric_motor_b200 import build as b; b.build()" > /dev/null
old=$(ls -td "$wt"/build/gemb200/*/ | head -1)
new=$(ls -td build/gemb200/*/ | head -1)
if [ "${2:-}" = "--per-function" ]; then python tools/sass_functions.py "$old" "$new" --all --skip-envp; exit $?; fi
sass() { cuobjdump -sass "$1" | sed 's#/\*[0-9a-f]*\*/##g' | grep -v '^identifier' | md5sum | cut -c1-16; }
shopt -s nullglob
status=0
for spec in host:1 step:12 jac:12 grad:12 psens:12; do
  kind=${spec%:*}; want=${spec#*:}
  same=0; diff=0
  for o in "$new$kind"*.o; do  # objects of the current build, and whether the reference build has the same SASS
    f=$(basename "$o")
    if [ -f "$old$f" ] && [ "$(sass "$old$f")" = "$(sass "$o")" ]; then same=$((same + 1)); else diff=$((diff + 1)); status=1; echo "DIFFERENT: $f"; fi
  done
  for o in "$old$kind"*.o; do  # objects only the reference build has
    f=$(basename "$o")
    if [ ! -f "$new$f" ]; then diff=$((diff + 1)); status=1; echo "MISSING in the current build: $f"; fi
  done
  if [ $((same + diff)) -ne "$want" ]; then status=1; echo "EXPECTED $want $kind objects, found $((same + diff))"; fi
  echo "$kind objects with identical SASS vs $ref: $same, different or missing: $diff"
done
exit $status
