#!/usr/bin/env bash
# A GPU session, stage by stage: what to run, in which order, with what time bound.  Every stage writes its log under
# gpurun_out/ (merged back by gpurun: keep it below 64 MiB - one `--set full --import-source on` report of 40 launches is
# already 47 MB; move old reports away first) and is wrapped in `timeout`, so a hang costs minutes, not the box.
# Usage (from the repo root, one stage list per gpurun call):
#     gpurun --timeout 1500 -- 'bash tools/gpu_round.sh tests bench'
#     gpurun --timeout 900  -- 'bash tools/gpu_round.sh ncu_set ncu_launches'
#     gpurun --gpus 2 --timeout 1200 -- 'bash tools/gpu_round.sh viewshard2'
#     gpurun --gpus 4 --timeout 900  -- 'NGPU=4 bash tools/gpu_round.sh nccl_tests strongN'
# Stages:
#   tests         the GPU suite (pytest -m gpu)
#   attn_poly     FMA-pipe exp2 variants of the spatial attention (V3D_ATTN_POLY=1..3): tests, then timings 0..3
#   micro_all     tools/microbench.py: every kernel family at its V3D_512 shapes
#   bench         bench.py (default N=1) -> gpurun_out/bench.json
#   bench_ref     bench.py --impl reference (host cores only, but the box time is charged all the same)
#   sweep         BASELINE configs[4]: S in {10,25,50} x T in {14,18,25} on one GPU -> gpurun_out/sweep.json
#   ncu_launches  the ncu launch list of one EDM step + decode (gpu__time_duration.sum, --clock-control none)
#   ncu_set       ONE ncu --set full run over every kernel family at its top-level shape (tools/microbench.py ncu_set)
#   ncu_full      ncu --set full of the named kernels inside bench.py (GEMM, attention, GroupNorm, LayerNorm)
#   viewshard2    (2 GPUs) the one-image-over-ranks parity tests, then the default line (image-parallel + `strong`) and
#                 the frame-sharded plan over torch.distributed collectives for comparison
#   nccl_tests    (NGPU GPUs) only the tests that need several GPUs
#   strongN       (NGPU GPUs) the default line: image-parallel value + `strong` (one image over the NGPU GPUs)
set -u
mkdir -p gpurun_out
PY=python
run() {  # run <seconds> <log> <cmd...>
  local t=$1 log=$2; shift 2
  echo "=== $* (timeout ${t}s) -> $log"
  timeout "$t" "$@" > "gpurun_out/$log" 2>&1
  local rc=$?
  echo "exit $rc" >> "gpurun_out/$log"
  tail -n 5 "gpurun_out/$log"
  return 0
}
for stage in "$@"; do
  case "$stage" in
    tests)
      run 1500 tests_gpu.log $PY -m pytest tests -m gpu -x -q ;;
    attn_poly)
      run 600 attn_poly_tests.log $PY -m pytest tests/test_kernels_gpu.py -m gpu -q -k "attention_poly_exp2"
      for k in 0 1 2 3; do V3D_ATTN_POLY=$k run 300 "micro_attn_poly$k.log" $PY tools/microbench.py attn; done ;;
    bench)
      run 900 bench.json $PY bench.py --steps 3 --warmup 3 ;;
    bench_ref)   # host cores only (charged GPU time all the same): run it sparingly
      run 900 bench_ref.json $PY bench.py --impl reference --steps 2 --warmup 1 ;;
    sweep)
      run 1500 sweep.log $PY tools/sweep.py ;;
    ncu_launches)
      V3D_CUDA_GRAPH=0 run 1200 ncu_launches.log ncu --metrics gpu__time_duration.sum --clock-control none -c 9000 --csv \
        --log-file gpurun_out/launches.csv $PY bench.py --steps 1 --warmup 0 --edm-steps 1 --no-cpu-baseline --no-parity ;;
    ncu_full)
      for k in gemm_tc_kernel attn_tc_kernel gn_stats_kernel gn_apply_kernel layernorm attn_temporal_kernel; do
        V3D_CUDA_GRAPH=0 run 600 "ncu_full_$k.log" ncu --set full --clock-control none --import-source on \
          -k "regex:$k" -s 40 -c 3 -o "gpurun_out/full_$k" -f $PY bench.py --steps 1 --warmup 0 --edm-steps 1 --no-cpu-baseline --no-parity
      done ;;
    ncu_set)
      # ONE ncu --set full run over every kernel family at its V3D_512 top-level shape (tools/microbench.py ncu_set)
      run 900 ncu_set.log ncu --set full --clock-control none --import-source on \
        -k "regex:gn_|layernorm|attn_|gemm_tc|softmax_rows" -c 40 -o gpurun_out/ncu_set -f $PY tools/microbench.py ncu_set ;;
    micro_all)
      run 600 micro_all.log $PY tools/microbench.py gemm conv attn norm small ;;
    viewshard2)
      # (2 GPUs) parity of the one-image-over-ranks plans (peer-memory transport by default over NCCL groups, then
      # torch.distributed collectives), then throughput: image-parallel line with its `strong` sub-object (all plans),
      # and the frame-sharded plan over NCCL collectives, eager and graph-captured, for comparison
      run 900 viewshard_tests.log $PY -m pytest tests/test_viewshard_gpu.py -m gpu -q -s -x
      run 900 bench_n2.json $PY -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29511 bench.py --gpus 2 --steps 3 --warmup 3
      V3D_SHARD_TRANSPORT=nccl run 900 bench_views2_nccl.json $PY -m torch.distributed.run --nnodes=1 --nproc-per-node 2 \
        --master-addr 127.0.0.1 --master-port 29512 bench.py --gpus 2 --shard views --steps 2 --warmup 3 --no-parity
      V3D_SHARD_TRANSPORT=nccl V3D_VIEWSHARD_GRAPH=1 run 900 bench_views2_nccl_graph.json $PY -m torch.distributed.run --nnodes=1 \
        --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29513 bench.py --gpus 2 --shard views --steps 2 --warmup 3 --no-parity ;;
    nccl_tests)
      run 700 viewshard_nccl_tests.log $PY -m pytest tests/test_viewshard_gpu.py -m gpu -q -s -x -k "nccl or cfg_views_engine_peer_transport" ;;
    strongN)
      # (N GPUs, N = $NGPU) the default line (image-parallel + `strong` sub-object)
      run 900 bench_n${NGPU:-8}.json $PY -m torch.distributed.run --nnodes=1 --nproc-per-node ${NGPU:-8} --master-addr 127.0.0.1 \
        --master-port 29521 bench.py --gpus ${NGPU:-8} --steps 3 --warmup 3 ;;
    *) echo "unknown stage $stage" ;;
  esac
done
