#!/bin/bash
# Round-end evidence, run under gpurun (1 GPU):
#   GPU tests, smoke, the default bench line (with CPU baseline, frame check and the config-5 extra),
#   the reference arm, the other workloads, ncu launch lists of the same commands and one
#   `--set full` capture of the top kernels per workload.
# Everything lands in the scratch output directory made below.
mkdir -p gpurun_out
R=${1:-r2}
python -m pytest tests -m gpu -q --timeout 600 2>&1 | tail -3 > gpurun_out/${R}_gpu_tests.txt
python -c "import __graft_entry__ as g; g.smoke()" >> gpurun_out/${R}_gpu_tests.txt 2>&1
python bench.py > gpurun_out/${R}_bench_paris4k.json 2> gpurun_out/${R}_bench_paris4k.err
python bench.py --impl reference --steps 10 --warmup 3 > gpurun_out/${R}_bench_reference_paris4k.json 2>/dev/null
for w in cubics100k circles8k paris4k_grad; do
  python bench.py --workload $w --no-cpu > gpurun_out/${R}_bench_$w.json 2>/dev/null
done
python bench.py --workload spaceship1080p --steps 100 --warmup 5 > gpurun_out/${R}_bench_spaceship1080p.json 2>/dev/null
for w in paris4k cubics100k circles8k; do
  ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file gpurun_out/${R}_launches_$w.csv \
      python bench.py --workload $w --steps 2 --warmup 1 --no-cpu --no-extra > /dev/null 2>&1
done
K='radix_downsweep_wide|radix_upsweep|radix_tile_scan|paint_kernel|cells_kernel|raster_emit|merge_entries|line_count'
ncu --set full --clock-control none --import-source on -k regex:"$K" -s 9 -c 9 -o gpurun_out/${R}_full_cubics100k -f \
    python bench.py --workload cubics100k --steps 2 --warmup 1 --no-cpu --no-extra > /dev/null 2>&1
ncu --set full --clock-control none --import-source on -k regex:'radix_downsweep_wide|radix_upsweep|paint_kernel|raster_emit|cells_kernel' \
    -s 7 -c 7 -o gpurun_out/${R}_full_paris4k -f python bench.py --workload paris4k --steps 2 --warmup 1 --no-cpu --no-extra > /dev/null 2>&1
ncu --set full --clock-control none --import-source on -k regex:'paint_kernel|radix_downsweep_wide' -s 4 -c 4 -o gpurun_out/${R}_full_circles8k -f \
    python bench.py --workload circles8k --steps 2 --warmup 1 --no-cpu --no-extra > /dev/null 2>&1
ls -la gpurun_out | grep ${R}_ | tail -30
