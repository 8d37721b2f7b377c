# End-of-round evidence: parity suite, bench lines for every workload, ncu launch list, timeline.
set -u
mkdir -p gpurun_out
timeout 300 python -m pytest tests -m gpu -x -q 2>&1 | tail -2 | tee gpurun_out/final_pytest.txt
timeout 60 python -c "import __graft_entry__ as g; g.smoke(); print('smoke ok')" 2>&1 | tail -1 | tee gpurun_out/final_smoke.txt
timeout 200 python bench.py 2>/dev/null | tail -1 > gpurun_out/final_bench_pcqm4m-small.json
timeout 200 python bench.py --impl reference 2>/dev/null | tail -1 > gpurun_out/final_bench_reference.json
for w in zinc-gine zinc-gatedgcn pcqm4m-medium-performer code2; do
  timeout 150 python bench.py --workload $w --steps 20 --warmup 3 2>/dev/null | tail -1 > gpurun_out/final_bench_$w.json
done
timeout 150 python bench.py --precision bf16 --steps 20 --warmup 3 2>/dev/null | tail -1 > gpurun_out/final_bench_pcqm4m-small_bf16.json
timeout 200 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file gpurun_out/final_launches.csv python bench.py --steps 2 --warmup 3 --no-graph > gpurun_out/final_ncu_bench.log 2>&1
timeout 120 python tools/profile_step.py pcqm4m-small > gpurun_out/final_timeline.txt 2>&1
