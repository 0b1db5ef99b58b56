#!/bin/bash
# usage: tools/run_scaling.sh <tag> [steps] [warmup] ["1 2 4 8"]   (run on a multi-GPU box; writes bench_out/scale_<tag>_*.json)
TAG=${1:-scale}; STEPS=${2:-300}; WARM=${3:-30}; NLIST=${4:-"1 2 4 8"}
mkdir -p bench_out
NG=$(python -c "import torch; print(torch.cuda.device_count())")
for MODE in lock hogwild; do
  for N in $NLIST; do
    [ "$N" -gt "$NG" ] && continue
    if [ "$N" = "1" ]; then
      timeout 300 python bench.py --gpus 1 --steps $STEPS --warmup $WARM --mode $MODE > bench_out/scale_${TAG}_${MODE}_$N.json 2> bench_out/scale_${TAG}_${MODE}_$N.err
    else
      timeout 300 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $((29600+N)) bench.py --gpus $N --steps $STEPS --warmup $WARM --mode $MODE > bench_out/scale_${TAG}_${MODE}_$N.json 2> bench_out/scale_${TAG}_${MODE}_$N.err
    fi
  done
done
python - <<PY
import json, glob, os
rows = []
for f in sorted(glob.glob("bench_out/scale_${TAG}_*.json")):
    txt = open(f).read().strip()
    if not txt: 
        print(f, "EMPTY", open(f.replace(".json", ".err")).read()[-400:]); continue
    d = json.loads(txt.splitlines()[-1])
    rows.append((d["config"]["parallelism"], d["n_gpus"], d["value"], d["ms_per_step"], d["e2e"]["value"], d["e2e"]["ms_per_step"], d["warm_cache_ms_per_step"]))
base = {}
for p, n, v, ms, ev, ems, wms in rows:
    mode = "lock" if "rw-lock" in p else "hogwild"
    if n == 1: base[mode] = (v, ev)
for p, n, v, ms, ev, ems, wms in rows:
    mode = "lock" if "rw-lock" in p else "hogwild"
    b = base.get(mode, (v, ev))
    print(f"{mode:8s} N={n}  dev {v/1e6:7.2f}M ({ms*1e3:6.1f}us, eff {v/(b[0]*n):.2f})  warm {wms*1e3:6.1f}us  e2e {ev/1e6:7.2f}M ({ems*1e3:6.1f}us, eff {ev/(b[1]*n):.2f})")
PY
