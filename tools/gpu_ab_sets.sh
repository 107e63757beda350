#!/bin/bash
# A/B several environment SETS of one build inside ONE gpurun call (box-to-box variance is ~5-10 %).
# usage: tools/gpu_ab_sets.sh "" "VLO_NO_PDL=1" ... [-- bench args]
set -u
SETS=()
while [ $# -gt 0 ] && [ "$1" != "--" ]; do SETS+=("$1"); shift; done
[ $# -gt 0 ] && shift
ARGS=${*:---steps 40 --warmup 5 --no-cpu-baseline}
for rep in 1 2; do
  for s in "${SETS[@]}"; do
    env $s timeout 300 python bench.py $ARGS 2>/dev/null | python -c "
import sys, json
for line in sys.stdin:
    try: d = json.loads(line)
    except Exception: continue
    ra = d.get('roofline_attn', {}); r = d.get('roofline', {}); ex = d.get('extras') or {}
    print('[$s]', 'value', round(d['value'],1), 'e2e', round(d['e2e']['value'],1), 'seq', round(d['config'].get('sequential_frames_per_s',0),1),
          'gemm_gbs', round(r.get('achieved',0)), 'attn_main_us', round(ra.get('main_kernel_only',{}).get('avg_us_per_launch',0),2),
          'ar_tok_s', round(ex.get('ar_decode',{}).get('tokens_per_s',0),1), 'ms8', round(ex.get('multistream8',{}).get('frames_per_s',0),1))
"
  done
done
