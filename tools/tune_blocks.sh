# diagnostic sweep of the launch-shape knobs of libb200pos.so (B2_TAIL_BLOCK, B2_DEC_BLOCK, B2_PAIRING_FORM) and the
# pipeline depth; run on the H100.  usage: bash tools/tune_blocks.sh "tail form depth [steps]" ...
[ $# -eq 0 ] && set -- "128 auto 3" "32 auto 3" "128 auto 4"
for cfg in "$@"; do
  set -- $cfg
  B2_TAIL_BLOCK=$1 B2_PAIRING_FORM=$2 timeout 300 python bench.py --steps ${4:-6} --warmup 3 --no-cpu-baseline --depth $3 2>/dev/null | python -c "
import sys, json
d = json.loads(sys.stdin.read().strip().splitlines()[-1])
st = d['stage_ms']
print('tail=$1 form=$2 depth=$3 steps=${4:-6}', 'pipelined', round(d['ms_per_step'],2), 'unpipelined', round(d['ms_per_step_unpipelined'],2), 'e2e', round(d['e2e']['ms_per_step'],2), 'agg', round(st['bls_aggregate_2^20_sigs'],2), 'fav', round(st['fast_aggregate_verify_2048'],2))
"
done
