#!/bin/bash
# One gpurun call, many answers: every call costs 1.5-3 minutes of box time before the command even starts, so measurements are
# batched.  Usage (from the repository root, on the GPU box):
#     bash tools/gpu_session.sh [tests] [smoke] [timeline] [variants] [p2gparts] [pcgparts] [overhead] [multi2] [barrier] [sanitize] [ncustep] [bench] [launches] [ncu] [blubrun]
# Everything lands in gpurun_out/session_*.{txt,json,csv}; nothing here is a bench number unless it comes from bench.py outside ncu.
set -u
OUT=gpurun_out
mkdir -p $OUT
want() { [[ " $ARGS " == *" $1 "* ]]; }
ARGS="${*:-tests timeline bench}"

if want tests; then         # the whole GPU suite, WITHOUT -x: every failure is listed
    timeout 900 python -m pytest tests -m gpu -q --tb=short -p no:cacheprovider 2>&1 | grep -v "^$" > $OUT/session_tests.txt
    tail -40 $OUT/session_tests.txt
fi
if want smoke; then         # twice: the round-1 failure was run-to-run
    for k in 1 2; do timeout 120 python -c "import __graft_entry__ as g; g.smoke()" > $OUT/session_smoke$k.txt 2>&1; tail -2 $OUT/session_smoke$k.txt; done
fi
if want timeline; then      # stage times over a dam break
    python tools/profile_targets.py stages dam_256 3 56 110 > $OUT/session_timeline_default.txt 2>&1
    python tools/profile_targets.py stages dam_halfhalf_highres 3 56 110 > $OUT/session_timeline_default_c3.txt 2>&1
    for f in default default_c3; do echo "== $f"; cat $OUT/session_timeline_$f.txt; done
fi
if want variants; then      # comparison paths against the default timeline
    BLUB_P2G=gather python tools/profile_targets.py stages dam_256 3 56 110 > $OUT/session_timeline_p2g_gather.txt 2>&1
    BLUB_PCG=tiles python tools/profile_targets.py stages dam_256 3 56 110 > $OUT/session_timeline_pcg_tiles.txt 2>&1
    python tools/profile_targets.py pcg 256 6 > $OUT/session_pcg_dense_default.txt 2>&1; cat $OUT/session_pcg_dense_default.txt
    for f in p2g_gather pcg_tiles; do echo "== $f"; grep -E "after|p2g|solve_|extrapolate |density_gather|total|Error|error" $OUT/session_timeline_$f.txt; done
fi
if want p2gparts; then      # which kernel of the P2G stage is slow late in the run: launch list of stage 0 at step 56 (eager launches) + cell statistics
    python tools/profile_targets.py cellstats dam_256 3 56 110 > $OUT/session_cellstats.txt 2>&1; cat $OUT/session_cellstats.txt
    BLUB_NO_GRAPH=1 timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -k regex:"cell_|scan_|marker_|p2g_" --launch-skip 566 -c 10 --csv \
        --log-file $OUT/session_p2g_parts.csv python tools/profile_targets.py step dam_256 58 > $OUT/session_p2g_parts.log 2>&1
    grep -v "^==" $OUT/session_p2g_parts.csv | python -c "
import csv,sys
for r in csv.DictReader(sys.stdin):
    if r.get('Metric Name')=='gpu__time_duration.sum': print(r['Kernel Name'][:60], r['Metric Value'], r['Metric Unit'])"
fi
if want pcgparts; then      # launch list of the solver kernels of one early step (eager launches)
    BLUB_NO_GRAPH=1 timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -k regex:"pcg_" --launch-skip 30 -c 12 --csv \
        --log-file $OUT/session_pcg_parts.csv python tools/profile_targets.py step dam_256 6 > $OUT/session_pcg_parts.log 2>&1
    grep -v "^==" $OUT/session_pcg_parts.csv | python -c "
import csv,sys
for r in csv.DictReader(sys.stdin):
    if r.get('Metric Name')=='gpu__time_duration.sum': print(r['Kernel Name'][:60], r['Metric Value'], r['Metric Unit'])"
fi
if want overhead; then
    python tools/profile_targets.py pcg_overhead > $OUT/session_pcg_overhead.txt 2>&1; cat $OUT/session_pcg_overhead.txt
fi
if want multi2; then        # needs gpurun --gpus 2: the multi-GPU tests, per-stage times of the sharded step, sanitizers on the 2-slab target
    timeout 600 python -m pytest tests/test_gpu_multi.py -m gpu -q --tb=short -p no:cacheprovider 2>&1 | grep -v "^$" | tail -30 > $OUT/session_multi_tests.txt; tail -12 $OUT/session_multi_tests.txt
    timeout 600 python tools/profile_targets.py stages_sharded 2 > $OUT/session_stages_sharded2.txt 2>&1; cat $OUT/session_stages_sharded2.txt
    SANITIZE_TIMEOUT=400 bash tools/sanitize.sh slab 2>&1 | tee $OUT/session_sanitize_slab.txt | tail -12
fi
if want barrier; then       # cost of one grid-wide sum, candidates in isolation (tools/barrier_bench.cu; built here if the binary did not travel)
    [ -x tools/barrier_bench ] || nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/barrier_bench tools/barrier_bench.cu
    ./tools/barrier_bench > $OUT/session_barrier.txt 2>&1; cat $OUT/session_barrier.txt
fi
if want sanitize; then
    bash tools/sanitize.sh pcg step 2>&1 | tee $OUT/session_sanitize.txt | tail -40
fi
if want ncustep; then       # full captures INSIDE the dam break (eager launches): the column solver at step 110, the P2G scatter + finish at step 5
    BLUB_NO_GRAPH=1 timeout 900 ncu --set full --clock-control none --import-source on -k regex:pcg_solve_columns --launch-skip 220 -c 1 -o $OUT/session_pcg_step110 \
        python tools/profile_targets.py step dam_256 111 > $OUT/session_ncu_pcg_step110.log 2>&1
    BLUB_NO_GRAPH=1 timeout 900 ncu --set full --clock-control none --import-source on -k regex:"p2g_scatter|p2g_normalize|marker_finalize|density_scatter|advect_kernel|correct_particles" --launch-skip 30 -c 6 -o $OUT/session_particle_kernels \
        python tools/profile_targets.py step dam_256 7 > $OUT/session_ncu_particles.log 2>&1
    ls -la $OUT/*.ncu-rep
fi
if want bench; then
    timeout 600 python bench.py > $OUT/session_bench.json 2> $OUT/session_bench.err
    head -c 600 $OUT/session_bench.json; echo; tail -3 $OUT/session_bench.err
fi
if want launches; then      # the launch list of the bench command itself (shares only: ncu serialises and runs cold)
    timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file $OUT/session_launches.csv \
        python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-roofline --no-scaling-reference --no-phases > $OUT/session_launches.log 2>&1
    python tools/summarize_ncu.py launches $OUT/session_launches.csv > $OUT/session_launches.md 2>&1; head -30 $OUT/session_launches.md
fi
if want ncu; then           # one full capture of the PCG kernel on the roofline microbench
    timeout 600 ncu --set full --clock-control none --import-source on -k regex:pcg_solve_columns -c 1 -o $OUT/session_pcg \
        python tools/profile_targets.py pcg 256 1 > $OUT/session_ncu.log 2>&1
    ls -la $OUT/session_pcg.ncu-rep
fi
if want blubrun; then
    ./blub_b200/blub_run tests/golden/scenes/dam_halfhalf.json --steps 320 --stats $OUT/session_run_stats.json --trace $OUT/session_run_trace.json > $OUT/session_run.txt 2>&1
    tail -2 $OUT/session_run.txt
fi
if want matchab; then       # warp aggregation of the scatter kernels: peer groups (match.any, default) against adjacent runs; cost of MATCH.ANY itself
    [ -x tools/match_bench ] || nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/match_bench tools/match_bench.cu
    ./tools/match_bench > $OUT/session_match_bench.txt 2>&1; cat $OUT/session_match_bench.txt
    BLUB_SCATTER_AGG=adjacent python tools/profile_targets.py stages dam_256 3 56 110 > $OUT/session_timeline_agg_adjacent.txt 2>&1
    echo "== adjacent runs"; grep -E "after|p2g|density_gather|advect|correct|binning|total|Error|error" $OUT/session_timeline_agg_adjacent.txt
    B="--steps 100 --warmup 10 --no-cpu-baseline --no-roofline --no-scaling-reference --no-phases"
    for v in "match 8" "adjacent 8" "match 12" "match 16" "match 4"; do
        set -- $v
        BLUB_SCATTER_AGG=$1 BLUB_RESORT_EVERY=$2 timeout 300 python bench.py $B > $OUT/session_bench_agg_$1_$2.json 2>> $OUT/session_bench.err
        python -c "import json,sys; d=json.load(open('$OUT/session_bench_agg_$1_$2.json')); print('agg $1 resort every $2:', d['value'], 'steps/s', d['ms_per_step'], 'ms, e2e', d['e2e']['value'])"
    done
fi
if want configs; then       # the other BASELINE configurations on one GPU (C2, C3, C5, C4), 100 steps after 10
    B="--steps 100 --warmup 10 --no-cpu-baseline --no-roofline --no-scaling-reference --no-phases"
    for w in dam_halfhalf dam_halfhalf_highres double_dam_box basin_512; do
        timeout 400 python bench.py --workload $w $B > $OUT/session_bench_$w.json 2>> $OUT/session_bench.err
        python -c "import json,sys; d=json.load(open('$OUT/session_bench_$w.json')); print('$w:', d['value'], 'steps/s', d['ms_per_step'], 'ms, e2e', d['e2e']['value'], d['config']['workload'], d['config']['particles'])"
    done
fi
if want ncuscatter; then    # full captures of the two scatter kernels at step 5, both aggregation forms (eager launches)
    for a in match adjacent; do
        BLUB_SCATTER_AGG=$a BLUB_NO_GRAPH=1 timeout 600 ncu --set full --clock-control none --import-source on -k regex:"p2g_scatter|density_scatter" --launch-skip 10 -c 2 -o $OUT/session_scatter_$a \
            python tools/profile_targets.py step dam_256 7 > $OUT/session_ncu_scatter_$a.log 2>&1
    done
    ls -la $OUT/session_scatter_*.ncu-rep
fi
if want multicheck; then    # needs gpurun --gpus 2: the multi-GPU tests and the N = 2 bench line (z-slab ranks run the same scatter kernels over their capacity)
    timeout 600 python -m pytest tests/test_gpu_multi.py -m gpu -q --tb=short -p no:cacheprovider 2>&1 | grep -v "^$" | tail -30 > $OUT/session_multi_tests.txt; tail -6 $OUT/session_multi_tests.txt
    timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29517 bench.py --gpus 2 --steps 20 --warmup 5 > $OUT/session_bench_n2.json 2> $OUT/session_bench_n2.err
    head -c 400 $OUT/session_bench_n2.json; echo; tail -3 $OUT/session_bench_n2.err
fi
if want pcgvariants; then   # in-step solve times of the comparison solvers (TMA-staged tiles, register-marching tiles) against the default column solver
    for v in tma tiles; do
        BLUB_PCG=$v python tools/profile_targets.py stages dam_256 3 56 110 > $OUT/session_timeline_pcg_$v.txt 2>&1
        echo "== BLUB_PCG=$v"; grep -E "after|solve_|total|Error|error" $OUT/session_timeline_pcg_$v.txt
    done
fi
