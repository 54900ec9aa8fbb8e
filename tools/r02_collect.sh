#!/bin/bash
# copies one measurement set (tools/r02_final.sh <tag>) from gpurun_out/ into profiles/ under stable names
set -u
tag=${1:?tag}; g=gpurun_out; p=profiles
head=$(git log -1 --format=%h)   # the snapshot the GPU box ran is this working tree (the box has no .git)
for c in C1 C1_reference C2 C3 C4; do [ -s $g/${tag}_bench_$c.json ] && tail -1 $g/${tag}_bench_$c.json > $p/r02_final_bench_$c.json; done
cp $g/${tag}_shape_sweep.log $p/r02_final_shape_sweep.log
cp $g/${tag}_launches.csv $p/r02_final_launches.csv
cp $g/${tag}_cli_feeds.log $p/r02_final_cli_feeds.log
cp $g/${tag}_logdecode_bench.log $p/r02_final_logdecode_bench.log
cp $g/${tag}_tests.log $p/r02_final_gpu_tests.log
for t in memcheck racecheck synccheck initcheck; do grep -E "ok|SUMMARY|Error|hazard" $g/${tag}_sanitizer_$t.log | head -20 > $p/r02_sanitizer_$t.log; done
cp $g/${tag}_sanitizer_summary.log $p/r02_sanitizer_summary.log
for m in hll alive counters; do
  python tools/ncu_summary.py $g/${tag}_prof_$m.ncu-rep $m $p/r02_final_${m}_ncu_summary.txt \
    "round 2 final, build $head: ncu --set full --clock-control none of kta::scan_kernel, bench.py --mode $m --tombstones 500 --steps 2 --warmup 1 (C1 shape, 1e8 records, one GPU)" > /dev/null
done
{
  echo "# SASS of the shipped libkta_gpu.so (build $head), cuobjdump -sass, scan_kernel<MODE_HLL, SMEM> = _ZN3kta11scan_kernelILi1ELb1ELb0ELb0EEEvNS_10ScanParamsE"
  f=$(mktemp)
  cuobjdump -sass -fun '_ZN3kta11scan_kernelILi1ELb1ELb0ELb0EEEvNS_10ScanParamsE' kafka_topic_analyzer_b200/libkta_gpu.so > $f 2>/dev/null
  grep -m1 "arch =" $f
  echo "# the key stage: bulk async copy global->shared (TMA engine, no tensor map) and its mbarrier"
  grep -E "UBLKCP|SYNCS" $f | sed 's/^\s*//'
  echo "# the tile loop's key reads, counter reductions and sketch raises (first of each kind)"
  for m in "LDS.128" "ATOMS.POPC.INC" "ATOMS.ADD" "REDUX" "RED.E.MAX" "LDG.E.*CONSTANT"; do grep -m2 -E "$m" $f | sed 's/^\s*//'; done
  echo "# mnemonic totals over the whole library (no UTMALDG / UTC*MMA / HMMA: there is no 2-D tile or contraction on this path)"
  cuobjdump -sass kafka_topic_analyzer_b200/libkta_gpu.so 2>/dev/null | grep -oE "\b(UBLKCP\.S\.G|SYNCS\.[A-Z0-9_.]+|ATOMS\.[A-Z0-9_.]+|C?REDUX[A-Z0-9_.]*|UTMALDG[A-Z0-9_.]*|UTC[A-Z]*MMA[A-Z0-9_.]*|HMMA[A-Z0-9_.]*|ATOMG\.[A-Z0-9_.]+|RED\.E\.[A-Z0-9_.]+)" | sort | uniq -c | sort -rn | head -30
  rm -f $f
} > $p/r02_final_sass_excerpt.txt
ls -la $p | grep r02_final
