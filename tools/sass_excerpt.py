#!/usr/bin/env python
"""SASS evidence per kernel of the shipped library: counts of the instructions that show how a kernel moves data
(UBLKCP = cp.async.bulk / TMA bulk copy, SYNCS = mbarrier, LDG.E.128 / LDS.128 / STS.128 = 128-bit accesses, VOTE = ballots),
plus a few lines of context around the first occurrence. Usage: python tools/sass_excerpt.py > profiles/r02_sass.md"""
import re, subprocess, sys, os, collections
LIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tuplex_b200", "lib", "libtplx_gpu.so")
out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
kern = None
data = collections.OrderedDict()
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        kern = subprocess.run(["c++filt", m.group(1)], capture_output=True, text=True).stdout.strip().split("(")[0]
        data[kern] = []
        continue
    m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
    if m and kern:
        data[kern].append(m.group(2).strip())
PAT = [("UBLKCP", r"UBLKCP"), ("SYNCS (mbarrier)", r"SYNCS"), ("LDG.E.128", r"LDG\.E\.128"), ("LDG.E.64", r"LDG\.E\.64"), ("LD.E (generic)", r"\bLD\.E"),
       ("LDS.128", r"LDS\.128"), ("STS.128", r"STS\.128"), ("LDS.64", r"LDS\.64"), ("STG.E.64", r"STG\.E\.64"), ("VOTE", r"VOTE"), ("ATOMG/RED", r"ATOMG|RED\.")]
want = [k for k in data if any(s in k for s in ("stage_mask", "stage_rows", "fused_scan_agg", "stage_hash", "mask_expand", "csv_parse_rows", "join_", "merge_", "valid_"))]
print("# SASS evidence (cuobjdump -sass tuplex_b200/lib/libtplx_gpu.so, sm_90a)\n")
print("| kernel | instructions | " + " | ".join(p[0] for p in PAT) + " |")
print("|---|---|" + "---|" * len(PAT))
for k in want:
    ins = data[k]
    print(f"| `{k}` | {len(ins)} | " + " | ".join(str(sum(1 for i in ins if re.search(p[1], i))) for p in PAT) + " |")
for k, pat in (("stage_mask_kernel<false>", r"UBLKCP|SYNCS"), ("stage_rows_vec_kernel<4>", r"LDG\.E\.128|LDS\.128|STS\.128"), ("fused_scan_agg_tma_kernel", r"UBLKCP")):
    kk = next((x for x in data if x.startswith("void tplx::" + k) or x.startswith("tplx::" + k) or k in x), None)
    if not kk:
        continue
    ins = data[kk]
    idx = [i for i, x in enumerate(ins) if re.search(pat, x)][:3]
    print(f"\n## `{kk}`: first occurrences of {pat}\n```")
    for i in idx:
        for x in ins[max(0, i - 2): i + 3]:
            print("    " + x)
        print("    ...")
    print("```")
