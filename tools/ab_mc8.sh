#!/bin/bash
# A/B of the gradient exchange modes at N GPUs (usage: tools/ab_mc8.sh N "mc pull"); short regions, no CPU arm
N=$1
for mode in $2; do
  D4PG_COMM_MODE=$mode timeout 300 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 2955$N bench.py --gpus $N --steps 2000 --warmup 20 --repeats 3 --no-cpu 2>${TMPDIR:-/tmp}/ab_mc_${N}_$mode.err | python -c "import json,sys; L=[x for x in sys.stdin if x.startswith('{')]; d=json.loads(L[-1]) if L else None; print('N=$N mode=$mode', (round(d['ms_per_step']*1e3,2), round(d['value']), d['replicas_identical'], d['implementation']['gradient_exchange'], round(d['e2e']['value'])) if d else 'FAILED')"
  tail -3 ${TMPDIR:-/tmp}/ab_mc_${N}_$mode.err
done
