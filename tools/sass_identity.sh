#!/bin/bash
# Is the device code of HEAD the same as that of commit $1?  Builds the 12 step translation units of that commit in a scratch worktree and
# compares `cuobjdump -sass` of every object with the current build (instruction addresses and the source-path identifier line removed).
#   bash tools/sass_identity.sh 503c048        (no GPU needed; ~1 min)
#   bash tools/sass_identity.sh 503c048 --per-function   kernel by kernel instead (tools/sass_functions.py), leaving out the ENVP
#        instantiations and reset_kernel, which share the objects with every other kernel
set -eu
ref=${1:?commit}
wt=$(mktemp -d /tmp/gemb200_sass_XXXX)
git worktree add -q "$wt" "$ref"
trap 'git worktree remove --force "$wt"' EXIT
(cd "$wt" && python -c "import sys; sys.path.insert(0, '$wt'); from gym_electric_motor_b200 import build as b; b.build(force=True, out='$wt/lib_ref.so')" > /dev/null)
python -c "from gym_electric_motor_b200 import build as b; b.build()" > /dev/null
old=$(ls -td "$wt"/build/gemb200/*/ | head -1)
new=$(ls -td build/gemb200/*/ | head -1)
if [ "${2:-}" = "--per-function" ]; then python tools/sass_functions.py "$old" "$new" --skip-envp; exit $?; fi
same=0; diff=0
for o in "$new"step_f*.o; do
  f=$(basename "$o")
  a=$(cuobjdump -sass "$old$f" | sed 's#/\*[0-9a-f]*\*/##g' | grep -v '^identifier' | md5sum | cut -c1-16)
  b=$(cuobjdump -sass "$o" | sed 's#/\*[0-9a-f]*\*/##g' | grep -v '^identifier' | md5sum | cut -c1-16)
  if [ "$a" = "$b" ]; then same=$((same + 1)); else diff=$((diff + 1)); echo "DIFFERENT: $f"; fi
done
echo "step translation units with identical SASS vs $ref: $same, different: $diff"
