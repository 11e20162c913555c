#!/bin/bash
# ncu captures and side checks; outputs go to the directory created below.
#   gpu_profile.sh ncu <kernel regex> <workload> [skip] [count]   full-set capture of a kernel of `bench.py --workload ...`
#   gpu_profile.sh launches <workload> [skip] [count]             launch list (gpu__time_duration) of the same command
#   gpu_profile.sh x3-timeline                                    per-layer timeline of conv_tower_x3_kernel
#   gpu_profile.sh two-gpu                                        multi-rank tests, 2-rank bench, 2-rank self-play entry point
mkdir -p gpurun_out
BENCH="python bench.py --steps 1 --warmup 3 --no-cpu-baseline --no-extras --no-loop --no-saturation"
case "$1" in
ncu)
    timeout 900 ncu --set full --clock-control none --import-source on -k "regex:$2" -s "${4:-4}" -c "${5:-1}" -o "gpurun_out/ncu_$2_$3" \
        $BENCH --workload "$3" > "gpurun_out/ncu_$2_$3.log" 2>&1; tail -2 "gpurun_out/ncu_$2_$3.log" | cut -c1-200 ;;
launches)
    timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -s "${3:-0}" -c "${4:-400}" --csv --log-file "gpurun_out/launches_$2.csv" \
        $BENCH --workload "$2" > "gpurun_out/launches_$2.log" 2>&1; ls -la "gpurun_out/launches_$2.csv" ;;
x3-timeline)
    rm -f gpurun_out/x3_timeline.txt
    MZ_NO_GRAPH=1 MZ_X3_TIMELINE=gpurun_out/x3_timeline.txt timeout 600 python scripts/x3_timeline.py | tee gpurun_out/x3_timeline.md ;;
two-gpu)
    timeout 600 python -m pytest tests -m gpu -q -x -k "rank or world or multi" 2>&1 | tail -4
    timeout 900 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 bench.py --gpus 2 --steps 20 --warmup 3 \
        > gpurun_out/bench_2gpu.json 2> gpurun_out/bench_2gpu.err; cut -c1-300 gpurun_out/bench_2gpu.json
    timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29512 -m muzero_general_b200.parallel \
        --game connect4 --games 2048 --reports 2 --moves-per-report 4 2>&1 | tail -3 ;;
*) sed -n 2,7p "$0" ;;
esac
