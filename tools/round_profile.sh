#!/bin/bash
# Round-end measurement set, run on the GPU box: tools/round_profile.sh TAG  (outputs under gpurun_out/)
TAG=${1:-r02}
O=gpurun_out
mkdir -p $O
KF='regex:caf_|wh_|metrics_|cfar_|det_|pl_|scan_|centroid_|compact_|interp_|fft_|spec_'
timeout 300 python -m pytest tests -x -q -m gpu 2>&1 | tail -3 > $O/${TAG}_pytest.log
python -c "import __graft_entry__ as g; g.smoke(); print('smoke ok')" >> $O/${TAG}_pytest.log 2>&1
timeout 200 python bench.py > $O/${TAG}_bench.json 2> $O/${TAG}_bench.err
timeout 120 python bench.py --steps 20 --warmup 5 --no-cpu-baseline > $O/${TAG}_bench_k20.json 2>> $O/${TAG}_bench.err
timeout 120 python bench.py --streams 1 --no-cpu-baseline > $O/${TAG}_bench_s1.json 2>> $O/${TAG}_bench.err
timeout 200 python bench.py --impl reference --steps 1 --warmup 0 > $O/${TAG}_bench_reference.json 2>> $O/${TAG}_bench.err
# launch list of the bench command (fewer steps: every launch is replayed by ncu; eager launches so that the list
# holds the steps' own launches and not the plan-creation runs of b200dd_pipeline_prepare_device)
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -k "$KF" -c 1500 --csv --log-file $O/${TAG}_launches_bench.csv \
    python bench.py --steps 6 --warmup 3 --no-cpu-baseline --eager > $O/${TAG}_ncu_bench.log 2>&1
# full sections: one cfg2 CPI (13 kernels) after two warm-up CPIs; one cfg3 CAF after two warm-up maps
timeout 200 ncu --set full --clock-control none --import-source on -k "$KF" --launch-skip 26 -c 13 -f -o $O/${TAG}_full_cfg2 \
    python tools/profile_target.py cfg2 3 > $O/${TAG}_ncu_cfg2.log 2>&1
timeout 200 ncu --set full --clock-control none --import-source on -k "regex:caf_range|caf_doppler" --launch-skip 4 -c 2 -f -o $O/${TAG}_full_cfg3 \
    python tools/profile_target.py cfg3 3 > $O/${TAG}_ncu_cfg3.log 2>&1
timeout 100 python tools/time_caf.py cfg1 cfg3 cfg4 > $O/${TAG}_time_caf.log 2>&1
timeout 60 python tools/wh_times.py > $O/${TAG}_wh_times.log 2>&1
timeout 100 python tools/bench_cfg5.py 5 2>/dev/null | tail -1 > $O/${TAG}_cfg5_n1.log
timeout 100 python tools/bench_cfg5.py 5 --no-filter 2>/dev/null | tail -1 >> $O/${TAG}_cfg5_n1.log
tools/ubench/fft64_dit > $O/${TAG}_fft64_dit.log 2>&1
tools/ubench/cvt_rates > $O/${TAG}_cvt_rates.log 2>&1
timeout 200 compute-sanitizer --tool racecheck --print-limit 20 tools/sanitize_native > $O/${TAG}_sanitizer_racecheck.log 2>&1
timeout 200 compute-sanitizer --tool memcheck --print-limit 20 tools/sanitize_native > $O/${TAG}_sanitizer_memcheck_native.log 2>&1
tail -2 $O/${TAG}_pytest.log; cut -c1-300 $O/${TAG}_bench.json; cut -c1-200 $O/${TAG}_bench_reference.json; tail -n 2 $O/${TAG}_ncu_cfg2.log; tail -n 2 $O/${TAG}_ncu_cfg3.log; tail -3 $O/${TAG}_sanitizer_racecheck.log; exit 0
