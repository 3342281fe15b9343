# Round evidence on one H100: the bench line (not under a profiler), the reference arm, the ncu launch list of the same
# bench command, one `ncu --set full` capture of the dominant kernel (the specialised fused Q1 pipeline) as CSV pages, its SASS,
# the operator table.  Everything lands in $OUT (small files).
set -x
OUT=gpurun_out/evidence; mkdir -p $OUT
R=${ROUND:-r02}
timeout 1500 python bench.py > $OUT/${R}_bench_n1.json 2> $OUT/${R}_bench_n1.err
timeout 600 python bench.py --impl reference > $OUT/${R}_bench_reference.json 2> $OUT/${R}_bench_reference.err
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file $OUT/${R}_launches_q1_bench.csv python bench.py --sf 20 --steps 3 --warmup 3 --skip-cpu --skip-e2e --skip-joins --skip-suites > $OUT/ncu_launches.log 2>&1
# launches of the specialised kernel in run_q1_once.py: one per repetition (the final aggregate and the sort are interpreted / small)
timeout 900 ncu --set full --import-source on --clock-control none -k regex:sg_jit_kernel --launch-skip 2 -c 1 -o /tmp/q1 python scripts/run_q1_once.py 10 4 > $OUT/ncu_q1.log 2>&1
ncu -i /tmp/q1.ncu-rep --page raw --csv > $OUT/${R}_q1_jit_kernel_raw.csv 2>/dev/null
ncu -i /tmp/q1.ncu-rep --page source --csv --print-source sass > /tmp/q1_source.csv 2>/dev/null
python scripts/ncu_sass_summary.py /tmp/q1_source.csv 50 > $OUT/${R}_q1_jit_kernel_sass_top.txt 2>&1
set +x
{ echo "# specialised kernels in sail_b200/_build/jit_cache after this run: resource usage (cuobjdump --dump-resource-usage), UBLKCP = TMA bulk copies, SYNCS = mbarrier instructions in the SASS"
  for f in sail_b200/_build/jit_cache/*.cubin; do echo "$(basename $f)  $(cuobjdump --dump-resource-usage $f | grep -oE "REG:[0-9]+ STACK:[0-9]+ SHARED:[0-9]+")  UBLKCP=$(cuobjdump -sass $f | grep -cE "UBLKCP") SYNCS=$(cuobjdump -sass $f | grep -cE "SYNCS")"; done; } > $OUT/${R}_jit_cubins.txt 2>&1
set -x
timeout 600 python scripts/bench_ops.py 10 > $OUT/ops.log 2>/dev/null; tail -1 $OUT/ops.log > $OUT/${R}_ops_sf10.json
timeout 1200 python scripts/bench_tpch.py 10 > $OUT/${R}_tpch_sf10.txt 2>&1
ls -la $OUT
