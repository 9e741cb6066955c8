#!/bin/bash
# The staged walker's traffic beside the haystack bytes, on one H100: the split copy model
# (profiles/microbench/stage_copy.cu), then this tree's library against the parent commit's, run alternately, and
# their outputs compared byte for byte.
#   scripts/gpu_feed_traffic.sh <checkout of the parent commit> [model] [flagship] [others]     (default: all three)
# (the checkout e.g. from `git archive HEAD~1 | tar -x -C <dir>`).  The libraries and the microbenchmark are built
# into build_variants/feed_traffic/ unless they are there already, so they can be built beforehand without a GPU.
# Reads the card's name and power limit; changes no setting and leaves nothing running.  Logs go to $OUT
# (default build_variants/feed_traffic/logs).
set -u
PARENT=${1:?a checkout of the parent commit}
shift
PARTS=${*:-model flagship others}
LIBS=build_variants/feed_traffic
OUT=${OUT:-$LIBS/logs}
mkdir -p $OUT $LIBS/parent $LIBS/cand
NVCC=${CUDA_HOME:-/usr/local/cuda}/bin/nvcc
FLAGS="-std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -diag-suppress 186 -shared -Xcompiler -fPIC,-pthread"
build() {  # <csrc dir> <library>: skipped when the library is already there (built beforehand, off the GPU)
  [ -f "$2" ] || $NVCC $FLAGS -o "$2" "$1/capi.cu" "$1/automaton.cpp" "$1/sieve.cpp" || exit 1
}
build "$PARENT/ahocorasick_rs_b200/csrc" $LIBS/parent/libacb200.so
build ahocorasick_rs_b200/csrc $LIBS/cand/libacb200.so
[ -x $LIBS/stage_copy ] || $NVCC -gencode arch=compute_90a,code=sm_90a -O3 -o $LIBS/stage_copy profiles/microbench/stage_copy.cu || exit 1

nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee $OUT/card.txt
case " $PARTS " in *" model "*) $LIBS/stage_copy | tee $OUT/stage_copy.txt ;; esac

bench() {  # <parent|cand> <log name> <bench.py arguments...>
  local which=$1 name=$2; shift 2
  ACB200_LIB=$PWD/$LIBS/$which/libacb200.so timeout 900 python bench.py --gpus 1 --no-cpu-baseline "$@" > $OUT/${which}_$name.json 2> $OUT/${which}_$name.err \
    || { echo "$which $name FAILED"; tail -5 $OUT/${which}_$name.err; return; }
  python - $OUT/${which}_$name.json $which $name <<'EOF'
import json, sys
d = json.loads(open(sys.argv[1]).read()); s = d["scan_stats"]
print(sys.argv[2], sys.argv[3], "ms/step %.4f" % d["ms_per_step"], "scan kernel ms %.4f" % d["roofline"]["kernel_ms"], "GB/s %.1f" % d["value"],
      "verified", d["verified"], "traps", s.get("traps"), "repairs", s.get("repairs"), "paths", s.get("paths"))
EOF
}
# 1. the flagship line, alternating, three times each
case " $PARTS " in *" flagship "*)
for i in 1 2 3; do
  for w in parent cand; do bench $w flag$i --config 2 --steps 2000 --warmup 5; done
done ;;
esac
case " $PARTS " in *" others "*) ;; *) exit 0 ;; esac
# 2. the other lines, once each, with what they returned
run_both() { local name=$1; shift; for w in parent cand; do bench $w $name "$@" --dump-outputs $OUT/dump_${w}_$name; done; }
run_both default --config 2 --steps 20 --warmup 5
run_both kernel3 --config 2 --steps 20 --warmup 5 --kernel 3
run_both table2 --config 2 --steps 20 --warmup 5 --table 2
run_both dense --config 2 --steps 20 --warmup 5 --dense --kernel 2
run_both config3 --config 3 --steps 200 --warmup 5
for name in default kernel3 table2 dense config3; do
  if diff -r $OUT/dump_parent_$name $OUT/dump_cand_$name > /dev/null; then echo "outputs $name: identical"; else echo "outputs $name: DIFFER"; fi
done
rm -rf $OUT/dump_parent_* $OUT/dump_cand_*
