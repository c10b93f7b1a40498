#!/bin/bash
# ncu captures on one GPU (never a multi-rank command): launch list of two steps, full captures of the dominant kernels.
# usage: tools/gpu_profile.sh [OUTPUT_DIR]   (default: profile_out)
OUT="${1:-profile_out}"
mkdir -p "$OUT"
B="python bench.py --steps 2 --warmup 3 --no-extras --no-cpu-baseline"
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 3000 --csv --log-file "$OUT/launches.csv" $B > "$OUT/ncu_launches.log" 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:"gemm_tc_kernel|attention_kernel|ln_stats_kernel|layernorm_kernel" -s 300 -c 9 -o "$OUT/encoder_full" $B > "$OUT/ncu_enc.log" 2>&1
timeout 900 ncu --set full --clock-control none --import-source on -k regex:"gemm_tc_kernel|topk_chunk_kernel|knn_rerank_kernel|embed_ln_kernel|sgemm_nt_kernel" -s 20 -c 8 -o "$OUT/knn_full" $B > "$OUT/ncu_knn.log" 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:"head_train_kernel" -s 1 -c 1 -o "$OUT/head_full" python tools/head_phase_times.py 20 > "$OUT/ncu_head.log" 2>&1
ls -la "$OUT"/*.ncu-rep "$OUT/launches.csv"
for f in enc knn head; do tail -n 2 "$OUT/ncu_$f.log"; done
