#!/bin/bash
# One-GPU evidence set (inside gpurun): isolated kernel table, ncu --set full captures of the top kernels, compute-sanitizer
# runs of the numerics self-tests, ncu launch list of three eager steps.  Everything lands in gpurun_out/.
O=gpurun_out
NCU="ncu --set full --clock-control none --import-source on -f"
timeout 240 python tools/profile_kernels.py --precision tf32 --iters 20 --out $O/kernels_tf32.json 2>&1 | tail -30
timeout 150 python tools/profile_kernels.py --precision bf16 --iters 20 --out $O/kernels_bf16.json 2>&1 | tail -3
timeout 200 $NCU -k regex:umma_gemm_kernel -s 3 -c 1 -o $O/prof_conv18_tf32 python tools/profile_kernels.py --precision tf32 --only conv18_fwd --iters 1 > $O/ncu_conv18_tf32.log 2>&1; echo "ncu conv18 rc=$?"
timeout 200 $NCU -k regex:linear_fwd_f32 -s 3 -c 1 -o $O/prof_linear50_fwd_f32 python tools/profile_kernels.py --precision tf32 --only linear_fwd_f32_4096x4096 --iters 1 > $O/ncu_linear50_fwd.log 2>&1; echo "ncu linear fwd rc=$?"
timeout 200 $NCU -k regex:linear_wgrad_f32 -s 3 -c 1 -o $O/prof_linear50_wgrad_f32 python tools/profile_kernels.py --precision tf32 --only linear50_wgrad_sgd_f32 --iters 1 > $O/ncu_linear50_wgrad.log 2>&1; echo "ncu linear wgrad rc=$?"
timeout 200 $NCU -k regex:conv_bn_act_p2p -s 3 -c 1 -o $O/prof_fused_cut7_tf32 python tools/profile_kernels.py --precision tf32 --only fused_cut7 --iters 1 > $O/ncu_fused_cut7_tf32.log 2>&1; echo "ncu fused rc=$?"
timeout 300 compute-sanitizer --tool memcheck --error-exitcode 9 python -m split_learning_b200.ops.selftest conv_fwd_tf32 conv_wgrad_tf32 fused_cut_tail_tf32 linear_f32 conv1_direct_f32 bn_fwd_bwd_f32 > $O/sanitizer_memcheck.log 2>&1; echo "memcheck rc=$?"; tail -4 $O/sanitizer_memcheck.log
timeout 300 compute-sanitizer --tool racecheck --error-exitcode 9 python -m split_learning_b200.ops.selftest linear_f32 conv1_direct_f32 bn_fwd_bwd_f32 > $O/sanitizer_racecheck.log 2>&1; echo "racecheck rc=$?"; tail -4 $O/sanitizer_racecheck.log
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -s 1400 -c 351 --csv --log-file $O/r2_launches_tf32_final.csv python bench.py --steps 6 --warmup 3 --no-graphs --no-api > $O/ncu_bench_final.log 2>&1; echo "launch list rc=$?"; wc -l $O/r2_launches_tf32_final.csv
