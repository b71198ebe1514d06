"""Extract the SASS of the key kernels from the built sm_90a extension into docs/sass/.

    python tools/dump_sass.py            # needs cuobjdump (CUDA toolkit); runs on the GPU-less build box
"""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "pytorch_distributed_b200", "_C.so")
OUT = os.path.join(ROOT, "docs", "sass")
WANT = {
    "fused_allreduce_bf16_nvls": r"fused_allreduce_kernelI13__nv_bfloat16Lb1E",
    "fused_allreduce_bf16_p2p": r"fused_allreduce_kernelI13__nv_bfloat16Lb0E",
    "oneshot_allreduce_f32_nvls": r"oneshot_allreduce_kernelIfLb1E",
    "fused_broadcast_f32_nvls": r"fused_broadcast_kernelIfLb1E",
    "reduce_to_caller_bf16_nvls": r"reduce_to_caller_kernelI13__nv_bfloat16Lb1E",
    "push_bf16_nvls": r"push_kernelI13__nv_bfloat16Lb1E",
    "metrics_bf16": r"metrics_kernelI13__nv_bfloat16E",
    "barrier": r"barrier_kernel",
    "fused_sgd_flat_bf16": r"fused_sgd_flat_kernelI13__nv_bfloat16S1_Lb1ELb0E",
    "gemm_bnstats_wgmma_n256": r"gemm_bnstats_kernelILi256E",
    "gemm_bnstats_wgmma_n64": r"gemm_bnstats_kernelILi64E",
    "combine_partials": r"combine_partials_kernel",
    "oneshot_allreduce_bf16_nvls": r"oneshot_allreduce_kernelI13__nv_bfloat16Lb1E",
    "stem_im2col": r"stem_im2col_kernelE",
    "stem_bwd_reduce_bf16": r"stem_bwd_reduce_kernelI13__nv_bfloat16E",
    "stem_fwd_bf16": r"stem_fwd_kernelI13__nv_bfloat16E",
    "stem_bwd_apply_bf16": r"stem_bwd_apply_kernelI13__nv_bfloat16E",
    "bn_stats_bf16": r"bn_stats_kernelI13__nv_bfloat16E",
    "bn_apply_bf16_relu_res": r"bn_apply_kernelI13__nv_bfloat16Lb1ELb1E",
    "bn_bwd_reduce_bf16_relu": r"bn_bwd_reduce_kernelI13__nv_bfloat16Lb1E",
    "bn_bwd_apply_bf16_relu_res": r"bn_bwd_apply_kernelI13__nv_bfloat16Lb1ELb1E",
    "bn_bwd_reduce_sum_bf16_relu": r"bn_bwd_reduce_sum_kernelI13__nv_bfloat16Lb1E",
}


def main():
    os.makedirs(OUT, exist_ok=True)
    txt = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", txt)
    summary = []
    for name, pat in WANT.items():
        hit = [f for f in funcs[1:] if re.search(pat, f.split("\n", 1)[0])]
        if not hit:
            summary.append("%-32s NOT FOUND (%s)" % (name, pat))
            continue
        body = hit[0].split("\nFatbin elf code")[0].rstrip() + "\n"      # the next translation unit's header is not part of it
        with open(os.path.join(OUT, name + ".sass"), "w") as f:
            f.write("Function : " + body)
        ops = re.findall(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]+)", body, flags=re.M)
        cnt = {}
        for o in ops:
            cnt[o] = cnt.get(o, 0) + 1
        key = [(k, v) for k, v in cnt.items() if re.match(r"(HGMMA|WARPGROUP|UTMA|SYNCS|LDGMC|STG\.E\..*SYS|LDG\.E\..*SYS|RED|ATOM|MULTIMEM|ST\.E\..*SYS|LD\.E\..*SYS|MEMBAR|CCTL|NANOSLEEP|BAR)", k)]
        summary.append("%-32s %5d instr; %s" % (name, len(ops), ", ".join("%s x%d" % kv for kv in sorted(key))))
    with open(os.path.join(OUT, "SUMMARY.txt"), "w") as f:
        f.write("SASS evidence (cuobjdump -sass pytorch_distributed_b200/_C.so, sm_90a). LDGMC = multimem.ld_reduce (in-switch reduce),\n"
                "STG/LDG ...STRONG.SYS = system-scope peer/multicast stores and loads, HGMMA = wgmma, UTMALDG / UTMASTG = TMA.\n\n")
        f.write("\n".join(summary) + "\n")
    print("\n".join(summary))


if __name__ == "__main__":
    sys.exit(main())
