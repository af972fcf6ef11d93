"""Committed SASS listings (BASELINE.json: "each shown in a committed SASS listing"): for every named hot kernel, the
instructions around its tensor-core mainloop (HGMMA = wgmma.mma_async, WARPGROUP = wgmma fences / wait_group, UTMALDG =
TMA, SYNCS = mbarrier) and its epilogue (peer ST / RED / ST.E.STRONG.SYS stores) cut out of ``cuobjdump -sass`` of the
in-tree library.

    python tools/sass_listings.py          # writes profiles/sass/*.sass + profiles/sass/README.md   (no GPU needed: cuobjdump only)
"""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "split_learning_b200", "ops", "_slb200.so")
DST = os.path.join(ROOT, "profiles", "sass")
KERNELS = {
    "conv_tf32_fwd_dgrad_bn64": "_ZN3slb16umma_gemm_kernelILi0ELi64EfLb0EEEv14CUtensorMap_stS1_NS_10GemmParamsE",
    "conv_tf32_wgrad_bn128": "_ZN3slb16umma_gemm_kernelILi1ELi128EfLb0EEEv14CUtensorMap_stS1_NS_10GemmParamsE",
    "conv_bf16_fwd_dgrad_bn64": "_ZN3slb16umma_gemm_kernelILi0ELi64E13__nv_bfloat16Lb0EEEv14CUtensorMap_stS2_NS_10GemmParamsE",
    "fused_cut_tail_tf32_bn64": "_ZN3slb22conv_bn_act_p2p_kernelILi64EfEEv14CUtensorMap_stS1_NS_14FusedCutParamsE",
    "fused_cut_tail_bf16_bn64": "_ZN3slb22conv_bn_act_p2p_kernelILi64E13__nv_bfloat16EEv14CUtensorMap_stS2_NS_14FusedCutParamsE",
    "fedavg_allreduce": "_ZN3slb23fedavg_allreduce_kernelENS_8ArParamsE",
    "linear_wgrad_sgd_f32": "_ZN3slb23linear_wgrad_f32_kernelEPKfS1_PfS2_S2_S2_S2_S2_iiiiiiiiiff",
    "sgd_momentum": "_ZN3slb19sgd_momentum_kernelEP6float4S1_S1_P5uint2xffi",
    "attn_fwd": "_ZN3slb15attn_fwd_kernelE14CUtensorMap_stS0_S0_NS_10AttnParamsE",
    "attn_bwd": "_ZN3slb15attn_bwd_kernelE14CUtensorMap_stS0_S0_S0_NS_10AttnParamsE",
    "linear_fwd_f32_ldgsts": "_ZN3slb21linear_fwd_f32_kernelEPKfS1_Pfiiiiiii",
    "linear_dgrad_f32_ldgsts": "_ZN3slb23linear_dgrad_f32_kernelEPKfS1_Pfiiiiiii",
    "ticket_publish": "_ZN3slb21ticket_publish_kernelEPjijjPKjj",
    "ticket_claim": "_ZN3slb19ticket_claim_kernelEPjijyPVj",
    "zero_wait_flag_acquire": "_ZN3slb16zero_wait_kernelEP6float4xPKjPjyPi",
    "litmus_pingpong": "_ZN3slb22litmus_pingpong_kernelEPjS0_PKjS2_ijiyS0_",
}
MARK = re.compile(r"HGMMA|WARPGROUP|UTMALDG|RED\.|REDG|ST\.E\.STRONG\.SYS|LD\.E\.STRONG\.SYS|SYNCS|MEMBAR|UTMAPF|ERRBAR|CCTL|LDGSTS|ATOM")


def listing(mangled):
    out = subprocess.run(["cuobjdump", "-sass", "-fun", mangled, LIB], capture_output=True, text=True).stdout
    lines = [l.rstrip() for l in out.splitlines() if re.search(r"/\*[0-9a-f]{4}\*/", l)]
    lines = [re.sub(r"\s*/\* 0x[0-9a-f]+ \*/\s*$", "", l) for l in lines]
    return lines


def main():
    os.makedirs(DST, exist_ok=True)
    readme = ["# SASS listings of the named hot kernels (sm_90a, `cuobjdump -sass split_learning_b200/ops/_slb200.so`)", "",
              "Each file holds the instruction windows around the tensor-core / TMA / mbarrier / peer-memory instructions of one kernel "
              "(full functions are thousands of lines; `tools/sass_listings.py` regenerates these from the in-tree library).", "",
              "| kernel | file | instructions | HGMMA | UTMALDG | WARPGROUP | SYNCS | RED | sys-scope ld/st | HMMA |", "|---|---|---:|---:|---:|---:|---:|---:|---:|---:|"]
    for name, mangled in KERNELS.items():
        lines = listing(mangled)
        if not lines:
            continue
        keep = set()
        for i, l in enumerate(lines):
            if MARK.search(l):
                keep.update(range(max(0, i - 3), min(len(lines), i + 4)))
        out, prev = [], -2
        for i in sorted(keep):
            if i != prev + 1:
                out.append("        ...")
            out.append(lines[i])
            prev = i
        demangled = subprocess.run(["c++filt", mangled], capture_output=True, text=True).stdout.strip()
        with open(os.path.join(DST, name + ".sass"), "w") as f:
            f.write(f"// {demangled}\n// {len(lines)} instructions; windows around wgmma / TMA / mbarrier / reduction / system-scope instructions\n")
            f.write("\n".join(out[:1200]) + "\n")
        txt = "\n".join(lines)
        c = lambda p: len(re.findall(p, txt))
        readme.append(f"| `{demangled[:90]}` | `{name}.sass` | {len(lines)} | {c('HGMMA')} | {c('UTMALDG')} | {c('WARPGROUP')} | {c('SYNCS')} | "
                      f"{c(r'RED[G.]')} | {c(r'STRONG.SYS')} | {c(r'\bHMMA')} |")
    open(os.path.join(DST, "README.md"), "w").write("\n".join(readme) + "\n")
    print("\n".join(readme))


if __name__ == "__main__":
    main()
