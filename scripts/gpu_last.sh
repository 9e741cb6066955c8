#!/bin/bash
# last look at the final tree on an H100: smoke and one short default bench line (stdout must be exactly one JSON line)
mkdir -p gpurun_out
python -c "import __graft_entry__ as g; g.smoke()" > gpurun_out/l_smoke.log 2>&1; tail -1 gpurun_out/l_smoke.log
timeout 100 python bench.py --steps 5 --warmup 3 --no-cpu-baseline > gpurun_out/l_bench.out 2> gpurun_out/l_bench.err; echo "bench rc=$? lines=$(wc -l < gpurun_out/l_bench.out)"
python -c "import json; d=json.loads(open('gpurun_out/l_bench.out').read()); print(d['value'], d['ms_per_step'], d['verified'], d['e2e']['value'])" || tail -5 gpurun_out/l_bench.err
