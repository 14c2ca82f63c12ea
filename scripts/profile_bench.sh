#!/bin/bash
# Run on a GPU machine (ONE GPU), writes under $OUT (default profile_out/): ncu launch list of the bench command + full captures of the kernels.
set -x
OUT="${OUT:-profile_out}"
mkdir -p "$OUT"
R=${1:-r02}
# (1) every launch with its device time (cold-cache, serialised: compare SHARES, not absolutes)
ncu --metrics gpu__time_duration.sum --clock-control none \
    -k regex:"sp_express|sp_encode|xxh3_chain|match_route|prep_rows|narrow_ids|assemble_segments|index_apply|index_insert|index_probe" \
    -c 400 --csv --log-file $OUT/${R}_launches.csv \
    python bench.py --requests 16384 --steps 2 --warmup 1 --no-cpu-baseline --no-c5 --no-latency --no-honest-text \
    > $OUT/${R}_launches_bench.log 2>&1
# (2) full capture of the tokenizer kernel at the bench's full size (one launch)
ncu --set full --clock-control none --import-source on -k regex:sp_express_kernel -s 2 -c 1 -o $OUT/${R}_sp_encode \
    python scripts/bench_encode.py --n 65536 --iters 1 --warmup 1 --check 0 > $OUT/${R}_ncu_sp.log 2>&1
# (3) full capture of the hash kernel at full size
ncu --set full --clock-control none --import-source on -k regex:xxh3_chain128 -s 3 -c 1 -o $OUT/${R}_xxh3 \
    python scripts/bench_hash.py --iters 1 > $OUT/${R}_ncu_xxh3.log 2>&1
# (4) full capture of the fused probe + scan + route kernel at the bench's size (64 Ki requests x 32 blocks, 1 Mi-key index)
ncu --set full --clock-control none --import-source on -k regex:match_route_kernel -s 3 -c 1 -o $OUT/${R}_match_route \
    python bench.py --steps 2 --warmup 3 --no-cpu-baseline --no-c5 --no-latency --no-honest-text \
    > $OUT/${R}_ncu_match.log 2>&1
for k in sp_encode xxh3 match_route; do
  python scripts/ncu_summary.py $OUT/${R}_${k}.ncu-rep > $OUT/${R}_${k}_ncu_full.txt 2>&1
done
python scripts/ncu_lines.py $OUT/${R}_sp_encode.ncu-rep > $OUT/${R}_sp_encode_lines.txt 2>&1
tail -2 $OUT/${R}_launches_bench.log | cut -c1-300
