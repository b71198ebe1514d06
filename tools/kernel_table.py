"""docs/KERNELS.md: one row per hand-written kernel (bf16 / NVLS instantiation) with the resources ptxas assigned.

    python tools/kernel_table.py          # needs cuobjdump; runs on the GPU-less build box against pytorch_distributed_b200/_C.so
"""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "pytorch_distributed_b200", "_C.so")

# (regex on the mangled name, display name, source, role, test or tool that checks it)
KERNELS = [
    (r"fused_allreduce_kernelI13__nv_bfloat16Lb1E", "fused_allreduce_kernel<bf16, NVLS>", "collectives.cu",
     "K1: pack + cast + 1/world + two-shot all-reduce (multimem.ld_reduce / multimem.st) (+ unpack); in-arena (bucket view) and single-rank variants", "tests/mp_gpu_checks.py, tools/comm_bench.py"),
    (r"fused_allreduce_kernelI13__nv_bfloat16Lb0E", "fused_allreduce_kernel<bf16, P2P>", "collectives.cu", "K1 over peer loads/stores (no multicast)", "tests/mp_gpu_checks.py"),
    (r"oneshot_allreduce_kernelI13__nv_bfloat16Lb1E", "oneshot_allreduce_kernel<bf16, NVLS>", "collectives.cu", "K1b: <= 512 KiB buckets: staging + ONE barrier + in-switch sum of the whole range into the arena", "tests/mp_gpu_checks.py"),
    (r"fused_broadcast_kernelIfLb1E", "fused_broadcast_kernel<fp32, NVLS>", "collectives.cu", "K2: weights / buffers from rank 0 (multicast store); deferred per-step BN-buffer broadcast", "tests/mp_gpu_checks.py"),
    (r"push_kernelI13__nv_bfloat16Lb1E", "push_kernel<bf16, NVLS>", "collectives.cu", "K2': DataParallel weight push", "tests/test_gpu_entrypoints.py"),
    (r"reduce_to_caller_kernelI13__nv_bfloat16Lb1E", "reduce_to_caller_kernel<bf16, NVLS>", "collectives.cu", "K5: in-switch gradient reduce onto GPU 0", "tests/test_gpu_entrypoints.py"),
    (r"metrics_kernelI13__nv_bfloat16E", "metrics_kernel<bf16>", "collectives.cu", "K4: top-1/top-5 counting + LL all-reduce of {loss, acc1, acc5}", "tests/test_gpu_kernels.py"),
    (r"ll_allreduce_kernel", "ll_allreduce_kernel", "collectives.cu", "<= 8 scalars, flag-in-payload protocol", "tests/mp_gpu_checks.py"),
    (r"barrier_kernel", "barrier_kernel", "collectives.cu", "K3", "tests/mp_gpu_checks.py"),
    (r"fused_sgd_flat_kernelI13__nv_bfloat16S1_Lb1ELb0E", "fused_sgd_flat_kernel<bf16 grad, bf16 model>", "optim.cu",
     "K6: unscale + overflow skip + SGD momentum over arena / fp32 masters / momentum / bf16 copy", "tests/test_gpu_kernels.py"),
    (r"fused_sgd_flat_kernelI13__nv_bfloat16S1_Lb1ELb1E", "fused_sgd_flat_kernel<bf16 grad, bf16 model, EMA>", "optim.cu",
     "K6 + --model-ema epilogue: fp32 weight average e = fmaf(d, e, w p) from the new masters", "tests/test_gpu_model_ema.py, tools/ema_bench.py"),
    (r"ema_multi_kernel", "ema_multi_kernel", "optim.cu", "--model-ema: BN buffers / stock-optimizer weights averaged, multi-tensor",
     "tests/test_gpu_model_ema.py, tools/ema_bench.py"),
    (r"grad_accumulate_kernel", "grad_accumulate_kernel", "collectives.cu",
     "--accum-steps: bucket gradients added into the rank-local fp32 sum (no_sync passes)", "tests/test_gpu_grad_accum.py, tools/accum_bench.py"),
    (r"grad_fold_kernel", "grad_fold_kernel", "collectives.cu",
     "--accum-steps: fp32 sum folded into the last pass's gradients and cleared, before K1", "tests/test_gpu_grad_accum.py, tools/accum_bench.py"),
    (r"fused_sgd_multi_kernel", "fused_sgd_multi_kernel", "optim.cu", "multi-tensor-apply variant (non-flat parameters)", "tests/test_gpu_kernels.py"),
    (r"larc_norm_flat_kernelI13__nv_bfloat16E", "larc_norm_flat_kernel<bf16>", "optim.cu",
     "LARC norm pass: per-chunk fp32 sums of p^2 and (g gmul)^2 over the arena, fixed order", "tests/test_gpu_larc.py, tools/larc_bench.py"),
    (r"larc_sgd_flat_kernelI13__nv_bfloat16S1_Lb1ELb0E", "larc_sgd_flat_kernel<bf16 grad, bf16 model>", "optim.cu",
     "LARC update: trust ratio from the chunk partials + SGD momentum + bf16 copy + statistics", "tests/test_gpu_larc.py, tools/larc_bench.py"),
    (r"larc_norm_multi_kernel", "larc_norm_multi_kernel", "optim.cu", "LARC norm pass, multi-tensor-apply variant", "tests/test_gpu_larc.py"),
    (r"larc_sgd_multi_kernel", "larc_sgd_multi_kernel", "optim.cu", "LARC update, multi-tensor-apply variant", "tests/test_gpu_larc.py"),
    (r"grad_sumsq_flat_kernelI13__nv_bfloat16E", "grad_sumsq_flat_kernel<bf16>", "optim.cu",
     "--clip-grad-norm norm pass: per-chunk fp32 sums of (g gmul)^2 over the arena's parameter ranges, LARC's order",
     "tests/test_gpu_clip_grad_norm.py, tools/clip_bench.py"),
    (r"grad_sumsq_multi_kernel", "grad_sumsq_multi_kernel", "optim.cu", "--clip-grad-norm norm pass, multi-tensor-apply variant",
     "tests/test_gpu_clip_grad_norm.py"),
    (r"clip_finalize_kernel", "clip_finalize_kernel", "optim.cu",
     "--clip-grad-norm: one CTA adds the partials in a fixed order, writes the norm, the clipped hyper copies and the count",
     "tests/test_gpu_clip_grad_norm.py, tools/clip_bench.py"),
    (r"multi_tensor_scale_kernel", "multi_tensor_scale_kernel", "optim.cu", "amp unscale with non-finite flag", "tests/test_gpu_kernels.py"),
    (r"amp_update_scale_kernel", "amp_update_scale_kernel", "optim.cu", "loss-scale state machine on the device", "tests/test_gpu_kernels.py"),
    (r"bn_stats_kernelI13__nv_bfloat16E", "bn_stats_kernel<bf16>", "bn_act.cu", "BN forward statistics (one row of partial sums per CTA)", "tests/test_gpu_kernels.py"),
    (r"bn_apply_kernelI13__nv_bfloat16Lb1ELb1E", "bn_apply_kernel<bf16, relu, res>", "bn_act.cu", "normalise + residual add + ReLU + 1-bit mask", "tests/test_gpu_kernels.py"),
    (r"bn_bwd_reduce_kernelI13__nv_bfloat16Lb1E", "bn_bwd_reduce_kernel<bf16, relu>", "bn_act.cu", "BN backward reductions", "tests/test_gpu_kernels.py"),
    (r"bn_bwd_apply_kernelI13__nv_bfloat16Lb1ELb1E", "bn_bwd_apply_kernel<bf16, relu, res>", "bn_act.cu", "dx, residual gradient, dgamma / dbeta", "tests/test_gpu_kernels.py"),
    (r"bn_bwd_reduce_sum_kernelI13__nv_bfloat16Lb1E", "bn_bwd_reduce_sum_kernel<bf16, relu>", "bn_act.cu", "add of two incoming gradients + mask + reductions (split residual gradients, default)", "tests/test_gpu_fused_paths.py"),
    (r"stem_fwd_kernelI13__nv_bfloat16E", "stem_fwd_kernel<bf16>", "bn_act.cu", "BN + ReLU + MaxPool 3x3/2 + arg-max codes", "tests/test_gpu_stem.py"),
    (r"stem_bwd_reduce_kernelI13__nv_bfloat16E", "stem_bwd_reduce_kernel<bf16>", "bn_act.cu", "stem backward reductions on 2x2 input quads", "tests/test_gpu_stem.py"),
    (r"stem_bwd_apply_kernelI13__nv_bfloat16E", "stem_bwd_apply_kernel<bf16>", "bn_act.cu", "stem backward apply", "tests/test_gpu_stem.py"),
    (r"gemm_bnstats_kernelILi256E", "gemm_bnstats_kernel<256>", "gemm_bnstats.cu",
     "wgmma / TMA 1x1-conv GEMM, BN statistics in the epilogue", "tests/test_gpu_tcgen05.py, tools/gemm_probe.py"),
    (r"gemm_bnstats_kernelILi64E", "gemm_bnstats_kernel<64>", "gemm_bnstats.cu", "same, N = 64 (also the stem GEMM)", "tests/test_gpu_tcgen05.py"),
    (r"combine_partials_kernel", "combine_partials_kernel", "bn_act.cu", "adds the per-CTA partial-sum rows of a reduction in a fixed order", "tests/test_gpu_kernels.py"),
    (r"stem_im2col_kernel", "stem_im2col_kernel", "stem_conv.cu", "7x7/2 patches of a C_in = 3 image as GEMM rows (v3: rows staged in shared memory)", "tests/test_gpu_fused_paths.py"),
    (r"normalize_kernelIh13__nv_bfloat16Li3ELb1E|normalize_kernelIf13__nv_bfloat16Li3ELb1E", "normalize_kernel<.., bf16, NHWC>", "data_ops.cu",
     "input normalise + cast + NCHW->NHWC", "tests/test_gpu_kernels.py"),
    (r"p2p_copy_kernel", "p2p_copy_kernel", "data_ops.cu", "multi-tensor peer copy (DataParallel gather)", "tests/test_gpu_misc.py"),
    (r"pack_only_kernelI13__nv_bfloat16", "pack_only_kernel<bf16>", "collectives.cu", "host-synchronised pack (single-process engine)", "tests/test_gpu_entrypoints.py"),
    (r"unpack_only_kernelI13__nv_bfloat16", "unpack_only_kernel<bf16>", "collectives.cu", "host-synchronised unpack (single-process engine)", "tests/test_gpu_entrypoints.py"),
    (r"multi_tensor_axpby_kernel", "multi_tensor_axpby_kernel", "optim.cu", "out = a*x + b*y over tensor lists (apex amp_C parity)", "tests/test_gpu_misc.py"),
]


def main():
    txt = subprocess.run(["cuobjdump", "-res-usage", SO], capture_output=True, text=True, check=True).stdout
    usage = {}
    name = None
    for line in txt.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+)", line)
        if m and name:
            usage[name] = tuple(int(g) for g in m.groups())
            name = None
    rows = []
    for pat, disp, src, role, ev in KERNELS:
        hit = [(k, v) for k, v in usage.items() if re.search(pat, k)]
        if not hit:
            rows.append("| `%s` | `csrc/%s` | %s | - | - | - | %s |" % (disp, src, role, ev))
            continue
        reg, stack, shared = hit[0][1]
        rows.append("| `%s` | `csrc/%s` | %s | %d | %d | %d | %s |" % (disp, src, role, reg, shared, stack, ev))
    out = os.path.join(ROOT, "docs", "KERNELS.md")
    with open(out, "w") as f:
        f.write("# Hand-written sm_90a kernels\n\n"
                "Generated by `tools/kernel_table.py` from `cuobjdump -res-usage pytorch_distributed_b200/_C.so` (nvcc 12.9, "
                "`-gencode arch=compute_90a,code=sm_90a -O3 --use_fast_math -lineinfo`).  Registers per thread, STATIC shared memory in bytes\n"
                "(the wgmma GEMM and the BN reductions add dynamic shared memory at launch), stack bytes.  The last column names the test\n"
                "(or tool) that checks the kernel; SASS excerpts: `tools/dump_sass.py` writes them to `docs/sass/`.\n\n"
                "| kernel | source | role | regs | smem | stack | evidence |\n|---|---|---|---:|---:|---:|---|\n")
        f.write("\n".join(rows) + "\n")
    print("wrote", out, "(%d kernels, %d found)" % (len(rows), sum(1 for r in rows if "| - |" not in r)))


if __name__ == "__main__":
    main()
