"""Instruction mix of a kernel's hottest loop from the SASS of libpysteps_b200.so:
    python tools/sass_count.py sl_multistep_kernelIfLb1ELb0
Finds the innermost backward branch with the largest body and counts its instructions by pipe."""
import re
import subprocess
import sys

so = "pysteps_b200/libpysteps_b200.so"
pat = sys.argv[1]
txt = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
funcs = re.split(r"\n\s*Function : ", txt)
body = next(f for f in funcs if pat in f.split("\n", 1)[0])
ins = []
for line in body.splitlines():
    m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
    if m:
        ins.append((int(m.group(1), 16), m.group(2).strip()))
addr = {a: i for i, (a, _) in enumerate(ins)}
loops = []
for i, (a, t) in enumerate(ins):
    m = re.search(r"\bBRA\b.*?0x([0-9a-f]+)", t)
    if m:
        tgt = int(m.group(1), 16)
        if tgt < a and tgt in addr:
            loops.append((addr[tgt], i))
print(f"{len(ins)} instructions, backward branches: {[(ins[s][0], ins[e][0], e - s + 1) for s, e in loops]}")
if not loops:
    sys.exit(0)
s, e = max(loops, key=lambda se: se[1] - se[0])
mix = {}
for _, t in ins[s:e + 1]:
    op = re.sub(r"^@!?U?P\d+\s+", "", t).split()[0].split(".")[0]
    mix[op] = mix.get(op, 0) + 1
fp64 = sum(v for k, v in mix.items() if k in ("DADD", "DMUL", "DFMA", "DSETP", "DMNMX"))
ld = sum(v for k, v in mix.items() if k.startswith("LD"))
print(f"largest loop body: {e - s + 1} instructions, FP64 pipe {fp64}, loads {ld}")
print(sorted(mix.items(), key=lambda kv: -kv[1]))
