#!/bin/bash
# Letterbox A/B in one command on the GPU: the card, the byte-stream ceilings (tools/lb_ceiling), the letterbox alone (tools/lb_probe.py)
# and the bench step, alternating a base library with the in-tree one.  The base library is another build of the same ABI
# placed at tensorrtx_b200/lib/libtrtx_hot_base.so (e.g. the parent commit's).  Everything lands in the directory given as the
# first argument (default lb_round_out/).
#   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/lb_ceiling tools/lb_ceiling.cu   (first)
set -u
OUT=${1:-lb_round_out}
export OUT
BASE=$PWD/tensorrtx_b200/lib/libtrtx_hot_base.so
mkdir -p $OUT
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee $OUT/card.txt
tools/lb_ceiling | tee $OUT/ceiling.log
TRTX_LIB=$BASE python tools/lb_probe.py > $OUT/probe.log
python tools/lb_probe.py >> $OUT/probe.log
for r in 1 2 3; do
    TRTX_LIB=$BASE python bench.py --steps 2000 --warmup 50 --no-cpu-baseline > $OUT/bench_base_$r.json 2>> $OUT/bench.err
    python bench.py --steps 2000 --warmup 50 --no-cpu-baseline > $OUT/bench_new_$r.json 2>> $OUT/bench.err
done
for c in retina_b16 v5s_b1; do
    for r in 1 2; do
        TRTX_LIB=$BASE python bench.py --config $c --steps 2000 --warmup 50 --no-cpu-baseline > $OUT/bench_${c}_base_$r.json 2>> $OUT/bench.err
        python bench.py --config $c --steps 2000 --warmup 50 --no-cpu-baseline > $OUT/bench_${c}_new_$r.json 2>> $OUT/bench.err
    done
done
# outputs at the timed size must not change
TRTX_LIB=$BASE python bench.py --steps 2000 --warmup 50 --no-cpu-baseline --dump-outputs $OUT/dump_base > /dev/null 2>> $OUT/bench.err
python bench.py --steps 2000 --warmup 50 --no-cpu-baseline --dump-outputs $OUT/dump_new > /dev/null 2>> $OUT/bench.err
python - <<'EOF'
import glob, json, os, statistics
import numpy as np
O = os.environ["OUT"]
for f in ("letterbox_sample", "detections"):
    a, b = np.load(f"{O}/dump_base/{f}.npy"), np.load(f"{O}/dump_new/{f}.npy")
    print(f, "array_equal:", a.shape == b.shape and np.array_equal(a, b))
for lib in ("libtrtx_hot_base.so", "libtrtx_hot.so"):
    for l in open(f"{O}/probe.log"):
        j = json.loads(l)
        if j["lib"] == lib:
            print("probe", lib, j["src"], j["out"], j["us"])
def runs(pat):
    return [json.load(open(f)) for f in sorted(glob.glob(f"{O}/{pat}"))]
for arm in ("base", "new"):
    rs = runs(f"bench_{arm}_[0-9].json")
    ms = [r["ms_per_step"] * 1e3 for r in rs]
    print(f"v8n_b32 {arm}: us/step {[round(x, 2) for x in ms]} median {statistics.median(ms):.2f}; letterbox us "
          f"{[round(r['kernels_us']['letterbox'], 2) for r in rs]}; scan us {[round(r['kernels_us']['scan'], 2) for r in rs]}; "
          f"clocks {rs[0]['clocks'].get('sm_mhz')} {rs[0]['clocks'].get('reasons')}")
for c in ("retina_b16", "v5s_b1"):
    for arm in ("base", "new"):
        rs = runs(f"bench_{c}_{arm}_[0-9].json")
        print(c, arm, "ms/step", [round(r["ms_per_step"], 4) for r in rs], "kernels_us", [r.get("kernels_us") for r in rs][:1])
EOF
timeout 900 python -m pytest -q -m gpu -p no:cacheprovider tests > $OUT/pytest_gpu.log 2>&1; echo "pytest gpu rc=$?"; tail -1 $OUT/pytest_gpu.log
python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -1
