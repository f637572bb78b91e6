"""Static SASS opcode histogram per kernel of libusdu_b200.so (what proves a Hopper-native kernel: UTMALDG / UTMASTG =
TMA bulk-tensor loads / stores, IMMA = mma.sync int8 tensor cores, I2IP = cvt.pack.sat, SYNCS / mbarrier traffic,
griddepcontrol = programmatic dependent launch).   python tools/sass_hist.py [out.json]"""
import collections
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "comfyui-distributed_b200", "libusdu_b200.so")
txt = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True).stdout
kern, hist = None, {}
for line in txt.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        # cut the parameter list only: "usdu::(anonymous namespace)::k(...)" keeps its namespace
        kern = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().rsplit("(", 1)[0]
        hist[kern] = collections.Counter()
        continue
    m = re.search(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)((?:\.[A-Z0-9_]+)*)", line)
    if m and kern:
        op = m.group(1)
        if op in ("IMMA", "HMMA", "LDG", "STG", "LDS", "STS", "ATOMS", "RED"):
            op += "".join(x for x in m.group(2).split(".")[:3] and ["." + p for p in m.group(2).split(".") if p in ("16832", "U8", "S8", "128", "64", "E")][:3])
        hist[kern][op] += 1
KEY = ("IMMA", "UTMALDG", "UTMASTG", "UTMAPF", "SYNCS", "I2IP", "PRMT", "IMAD", "SHFL", "LDS", "STS", "LDG", "STG", "F2I", "ACQBULK", "GRIDDEP")
out = {}
for k, c in hist.items():
    if not any(s in k for s in ("mma::", "fast::", "usdu::")):
        continue
    row = {"total": sum(c.values())}
    for key in KEY:
        n = sum(v for op, v in c.items() if op.startswith(key))
        if n:
            row[key] = n
    out[k] = row
js = json.dumps(out, indent=1)
if len(sys.argv) > 1:
    open(sys.argv[1], "w").write(js)
print(js)
