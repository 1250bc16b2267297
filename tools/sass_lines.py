"""Static SASS instructions per source line of one kernel (needs -lineinfo):  python tools/sass_lines.py <obj> <mangled-substring> [top]
Shows where a kernel's code volume is, without a GPU."""
import collections
import re
import subprocess
import sys

obj, pat = sys.argv[1], sys.argv[2]
top = int(sys.argv[3]) if len(sys.argv) > 3 else 40
import glob
import os
import tempfile

tmp = tempfile.mkdtemp()
subprocess.run(["cuobjdump", "-xelf", "all", os.path.abspath(obj)], cwd=tmp, stdout=subprocess.DEVNULL)
out = "".join(subprocess.run(["nvdisasm", "-g", "-c", c], stdout=subprocess.PIPE, text=True).stdout for c in glob.glob(tmp + "/*.cubin"))
cnt = collections.Counter()
on = False
line = None
total = 0
for l in out.splitlines():
    m = re.match(r"\s*\.section\s+\.text\.(\S+?),", l)
    if m:
        on = pat in m.group(1)
        continue
    if not on:
        continue
    m = re.search(r'//## File "([^"]+)", line (\d+)', l)
    if m:
        line = (m.group(1).split("/")[-1], int(m.group(2)))
        continue
    if re.match(r"\s+/\*[0-9a-f]{4}\*/\s+\S", l):
        cnt[line] += 1
        total += 1
print("total static", total)
src = {}
for (f, n), c in cnt.most_common(top):
    if f not in src:
        try:
            src[f] = open("gym_electric_motor_b200/csrc/" + f).read().splitlines()
        except OSError:
            src[f] = []
    text = src[f][n - 1].strip()[:110] if 0 < n <= len(src[f]) else ""
    print(f"{c:5d}  {f}:{n}  {text}")
