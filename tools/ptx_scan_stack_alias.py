"""Scan the PTX of csrc/b2s_capi.cu for the code-generation hazard that hid the EPA bug of round 1: two different pointer
arguments of one call that resolve to the SAME stack offset (nvcc 12.9 merged the stack slots of a direction vector and its
negation, so a callee received the same array twice).  usage: python tools/ptx_scan_stack_alias.py  (CPU only, needs nvcc)"""
import os, re, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ptx = os.path.join(tempfile.mkdtemp(), "b2s.ptx")
subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-ptx", "-o", ptx,
                       os.path.join(ROOT, "robosuite_b200", "csrc", "b2s_capi.cu")])
txt = open(ptx).read()
funcs = re.split(r"\n(?=\.(?:visible |weak )?(?:func|entry))", txt)
sus = 0
for f in funcs:
    m = re.match(r"\.(?:visible |weak )?(?:func|entry)\s*(?:\([^)]*\)\s*)?(\S+?)\(", f)
    name = m.group(1) if m else "?"
    defs = {}
    for r, base, k in re.findall(r"add\.u64\s+(%rd\d+), (%SPL?), (\d+);", f):
        defs.setdefault(r, set()).add(int(k))
    for call in re.findall(r"\{ // callseq.*?\} // callseq", f, flags=re.S):
        seen = {}
        for p, r in re.findall(r"st\.param\.b64\s+\[param(\d+)\], (%rd\d+);", call):
            if r in defs and len(defs[r]) == 1:
                k = next(iter(defs[r]))
                if k in seen and seen[k][1] != r:
                    print("same stack offset %d passed as params %s and %s in %s" % (k, seen[k][0], p, name[:80]))
                    sus += 1
                seen[k] = (p, r)
print("functions: %d, call sites passing one stack offset as two pointer arguments: %d" % (len(funcs), sus))
# Review aid for the round-1 case itself (the two arrays went to two CONSECUTIVE calls, which no per-call check can see):
# functions in which one stack offset is materialised under several registers.  Legitimate slot sharing looks the same, so
# these are the functions whose device-vs-oracle parity tests deserve a second look after a compiler upgrade.
shared = 0
for f in funcs:
    m = re.match(r"\.(?:visible |weak )?(?:func|entry)\s*(?:\([^)]*\)\s*)?(\S+?)\(", f)
    by = {}
    for r, k in re.findall(r"add\.u64\s+(%rd\d+), %SPL, (\d+);", f):
        by.setdefault(int(k), set()).add(r)
    multi = {k: len(v) for k, v in by.items() if len(v) > 1}
    if multi:
        shared += 1
        print("  shared-offset registers in %s: %s" % ((m.group(1) if m else "?")[:70], multi))
print("functions with shared-offset registers: %d" % shared)
sys.exit(1 if sus else 0)
