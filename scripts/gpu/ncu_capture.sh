#!/bin/bash
# ONE-GPU ncu captures of the multi-rank kernels (ranks emulated in-process, flags pre-signalled, one kernel at a time:
# "peer" accesses hit local HBM, so these show instruction mix / occupancy / memory-pipe behaviour, not NVLink) plus the
# single-GPU kernels. Run under gpurun. Each report holds 1-4 launches so that everything fits gpurun's 64 MiB return
# limit; CSV summaries are also produced ON the box (gpurun_out/ncu_csv/) in case the reports do not make it back.
set -x
cd "$(dirname "$0")/../.."
mkdir -p gpurun_out/ncu gpurun_out/ncu_csv
NCU="ncu --set full --clock-control none --import-source on"
# FT-ZeRO-1 big kernels at W=8 (rank 0's launches: reduce over a 256 MB unit, update of its 2 held slices)
$NCU -k regex:'zero1_(reduce|update)_kernel' -s 1 -c 2 -o gpurun_out/ncu/zero1_w8 -f \
  python bench/zero1_bench.py --virtual 8 --mb 256 --iters 1 --warmup 1 > gpurun_out/ncu/zero1_w8.log 2>&1
# world-1 update (= the flagship's AdamW at N=1)
$NCU -k regex:'zero1_update_kernel' -s 11 -c 1 -o gpurun_out/ncu/zero1_update_w1 -f \
  python bench/kernel_micro.py --only zero1_update --iters 1 > gpurun_out/ncu/micro_a.log 2>&1
$NCU -k regex:'diloco_outer_kernel' -s 3 -c 1 -o gpurun_out/ncu/diloco_outer -f \
  python bench/kernel_micro.py --only diloco_outer --iters 1 > gpurun_out/ncu/micro_b.log 2>&1
$NCU -k regex:'heal_copy_kernel' -s 11 -c 1 -o gpurun_out/ncu/heal_copy_lsu -f \
  python bench/kernel_micro.py --only heal_copy --iters 1 > gpurun_out/ncu/micro_c.log 2>&1
# the q8 large-message pipeline and the generic collectives (W=4 in-process, presignalled)
$NCU -k regex:'q8_|reduce_scatter_kernel|push_exchange' -c 6 -o gpurun_out/ncu/collectives -f \
  python -c "import torch; torch.cuda.set_device(0); from torchft_b200.bench_utils import collectives_selfcheck as c; print(c(world=4, nelem=1<<22))" > gpurun_out/ncu/selfcheck.log 2>&1
python scripts/ncu_summarize.py gpurun_out/ncu/*.ncu-rep --out gpurun_out/ncu_csv > gpurun_out/ncu/summarize.log 2>&1
# launch list of smoke() as the driver sees it
ncu --metrics gpu__time_duration.sum --clock-control none -c 600 --csv --log-file gpurun_out/ncu_csv/smoke_launches.csv \
  python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/ncu/smoke.log 2>&1
du -sh gpurun_out/ncu gpurun_out/ncu_csv
# keep the return under the limit: drop the largest reports first if needed (their CSV summaries stay)
while [ "$(du -sm gpurun_out | cut -f1)" -gt 48 ]; do
  big=$(ls -S gpurun_out/ncu/*.ncu-rep 2>/dev/null | head -1); [ -z "$big" ] && break; rm -f "$big"
done
ls -la gpurun_out/ncu gpurun_out/ncu_csv
