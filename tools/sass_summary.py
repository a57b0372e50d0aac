#!/usr/bin/env python
"""Opcode census of the shipped sm_90a kernels (cuobjdump -sass): writes profiles/sass_<kernel>.txt (full SASS of
the kernels DESIGN.md discusses) and prints a table of the opcodes that matter for the Hopper evidence: DMMA (fp64
tensor core), DFMA, UBLKCP / LDGSTS (bulk and per-thread async copies), SYNCS (mbarrier), RED / ATOM, LDG / STG widths.
    python tools/sass_summary.py            # after __graft_entry__.build()
"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBS = {"libdynoba.so": ["linearize_kernel<5", "schur_accum_kernel<2", "schur_stage_kernel<2", "band_cholesky_dataflow_kernel_v3", "band_backward_cluster_kernel",
                        "flow_pose_kernel", "motion_refine_kernel"],
        "libdynofront.so": ["klt_kernel", "sc_count_kernel", "pm_warp_kernel"]}
CENSUS_ONLY = ("flow_pose_kernel", "motion_refine_kernel")
KEYS = ["DMMA", "DFMA", "DADD", "DMUL", "MUFU", "UBLKCP", "LDGSTS", "SYNCS", "RED", "ATOM", "LDG.E.64", "LDG.E.128", "LDG.E.U8", "LDG.E ", "STG.E.64", "STG.E.128",
        "STG.E ", "LDS", "STS", "LDL", "STL", "BAR", "SHFL", "UTMALDG", "HGMMA"]

def demangle(n):
    try:
        return subprocess.run(["c++filt", n], capture_output=True, text=True).stdout.strip()
    except Exception:
        return n

def main():
    rows = []
    for lib, wanted in LIBS.items():
        path = os.path.join(ROOT, "dynosam_b200", lib)
        sass = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True).stdout
        blocks = re.split(r"\n\s*Function : ", sass)[1:]
        for b in blocks:
            name = demangle(b.split("\n", 1)[0].strip())
            hit = [w for w in wanted if w in name.replace(", ", ",").replace("> ", ">")]
            if not hit and not any(w.split("<")[0] in name and "<" in w and w in name.replace(" ", "") for w in wanted):
                continue
            ops = collections.Counter()
            n_inst = 0
            for line in b.split("\n"):
                m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
                if not m:
                    continue
                n_inst += 1; op = m.group(2)
                for k in KEYS:
                    if op.startswith(k.strip()) and (not k.endswith(" ") or op == k.strip()):
                        ops[k.strip() if not k.endswith(" ") else k.strip() + " (32-bit)"] += 1
            short = re.sub(r"\(.*", "", name).replace("dynoba::", "")
            fn = os.path.join(ROOT, "profiles", "sass_" + re.sub(r"[^A-Za-z0-9]+", "_", short).strip("_") + ".txt")
            if not any(w in name for w in CENSUS_ONLY):           # large scalar kernels: census row only, no multi-MB dump in the repo
                os.makedirs(os.path.dirname(fn), exist_ok=True)
                open(fn, "w").write(f"// cuobjdump -sass {lib}, function {name}\n" + b)
            rows.append((lib, short, n_inst, ops))
    print("| kernel | instructions | " + " | ".join(k.strip() for k in KEYS) + " |")
    print("|---|---|" + "---|"*len(KEYS))
    for lib, short, n, ops in rows:
        print(f"| `{short}` | {n} | " + " | ".join(str(ops.get(k.strip() if not k.endswith(' ') else k.strip() + ' (32-bit)', 0)) for k in KEYS) + " |")

if __name__ == "__main__":
    main()
