#!/bin/bash
# A/B of kernel variants selected by environment switches, on the benchmark configuration (no CPU arm, no Step-2 legs):
#   tools/ab_bench.sh "label1:ENV1=a ENV2=b" "label2:" ...
for spec in "$@"; do
  label="${spec%%:*}"; envs="${spec#*:}"
  env $envs timeout 200 python bench.py --no-cpu --no-step2 --steps 5 2>gpurun_out/ab_err.txt | python -c "
import json,sys
t=sys.stdin.read().strip().splitlines()
if t:
    j=json.loads(t[-1]); k=j.get('kernels',{})
    print('%-28s ms/step %6.2f  (%.0f SNPs/s, e2e %.0f)  single-lane ms/50 blocks: predict %.1f mx %.1f gram %.1f stats %.1f' % ('$label', j['ms_per_step'], j['value'], j.get('e2e',{}).get('value',0), k.get('l0_predict',{}).get('ms_total',0), k.get('mx_solve',{}).get('ms_total',0), k.get('gram_wgmma',{}).get('ms_total',0), k.get('l0_stats',{}).get('ms_total',0)))
else:
    print('%-28s failed: ' % '$label', open('gpurun_out/ab_err.txt').read()[-300:])"
done
