#!/usr/bin/env python
"""Full SASS listings (cuobjdump -sass) of the kernels the north star names, one file per kernel under OUT/sass/, plus a mnemonic
summary (OUT/sass_summary.txt), from the objects of the in-tree build.  Needs no GPU:  python benchmarks/dump_sass.py OUT"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "deeprec_b200", "lib", "obj")
WANT = {  # object file -> kernel-name substrings to dump in full
    "sparse_pipeline.cu.o": ["k_sp_dedup", "k_sp_lookupILi4", "k_sp_segsumILi4", "k_sp_gradILi4", "k_sp_gatherILi4", "k_sp_reset"],
    "comm_kernels.cu.o": ["k_allreduce_apply", "k_rank_barrier"],
    "fused_interaction_gemm.cu.o": ["k_dlrm_inter_gemm"],
    "interaction_kernels.cu.o": ["k_dot_fwd_tcILb1", "k_dot_bwd_tcILb1"],
    "gemm_wgmma.cu.o": ["k_gemm_tnILi128ELb0ELb0ELb0ELb0", "k_gemm_tnILi128ELb0ELb1ELb0ELb0", "k_gemm_tnILi64ELb0ELb0ELb1ELb1",
                        "k_gemm_nt_splitkILi128"],
    "tier_kernels.cu.o": ["k_tier_miss_list", "k_tier_evict"],
    "nvls.cu.o": ["k_nvls_allreduce_apply", "k_nvls_reduce_bcast"],
}
KEY = ["HGMMA", "QGMMA", "WARPSYNC", "HMMA", "LDGMC", "LDTM", "STTM", "UTMALDG", "UTMASTG", "UBLKCP", "SYNCS", "ACQBULK", "REDG", "ATOMG", "ATOMS", "MATCH", "LDG", "STG", "MEMBAR", "CCTL", "ERRBAR"]


def main():
    if len(sys.argv) != 2:
        raise SystemExit("usage: python benchmarks/dump_sass.py OUT")
    out_root = sys.argv[1]
    out_dir = os.path.join(out_root, "sass")
    os.makedirs(out_dir, exist_ok=True)
    summary = ["# SASS mnemonic counts per kernel (cuobjdump -sass of deeprec_b200/lib/obj/*.o, sm_90a); full listings of the starred kernels in sass/",
               "# HGMMA = wgmma bf16, QGMMA = wgmma e4m3, HMMA = mma.sync, UTMALDG/UTMASTG = TMA load/store, SYNCS = mbarrier, REDG = red.global,",
               "# MATCH = match.any, UCGABAR_ARV = barrier.cluster.arrive,",
               "# LDG/STG with .SYS or on peer-mapped pointers + MEMBAR.SC.SYS / ld.acquire.sys (LDG.E.STRONG.SYS) = in-kernel NVLink signalling", ""]
    for obj in sorted(os.listdir(OBJ)):
        if not obj.endswith(".o"):
            continue
        txt = subprocess.run(["cuobjdump", "-sass", os.path.join(OBJ, obj)], capture_output=True, text=True).stdout
        funcs = re.split(r"\n\s*Function : ", txt)[1:]
        for f in funcs:
            name = f.split("\n", 1)[0].strip()
            body = f
            ops = collections.Counter()
            for line in body.splitlines():
                m = re.match(r"\s*/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
                if m:
                    ops[m.group(1).split(".")[0]] += 1
                    if ".SYS" in m.group(1):
                        ops["*.SYS"] += 1
            short = subprocess.run(["c++filt", name], capture_output=True, text=True).stdout.strip() or name
            short = re.sub(r"\(anonymous namespace\)::", "", short).split("(")[0]
            star = any(w in name for w in WANT.get(obj, []))
            keyc = ", ".join(f"{k}={ops[k]}" for k in KEY + ["*.SYS", "UCGABAR_ARV"] if ops.get(k))
            summary.append(f"{'*' if star else ' '} {obj[:-5]:28s} {short[:70]:70s} instrs={sum(ops.values()):6d}  {keyc}")
            if star:
                fn = re.sub(r"[^A-Za-z0-9_]+", "_", short)[:80] + ".sass"
                lines = []
                for line in body.splitlines():
                    if re.match(r"\s*/\* 0x[0-9a-f]+ \*/\s*$", line):
                        continue                                   # second half of the 128-bit encoding
                    lines.append(re.sub(r"\s*/\* 0x[0-9a-f]+ \*/\s*$", "", line).rstrip())
                with open(os.path.join(out_dir, fn), "w") as fh:
                    fh.write(f"// {short}\n// {obj}  (nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo); encodings stripped\n\tFunction : " + "\n".join(lines) + "\n")
    with open(os.path.join(out_root, "sass_summary.txt"), "w") as fh:
        fh.write("\n".join(summary) + "\n")
    print("\n".join(l for l in summary if l.startswith("*")))


if __name__ == "__main__":
    main()
