#!/bin/bash
# Build cycle-accounting libraries (-DQPB_TIMING) for scripts/phase_timing.py, which loads one with QPB200_TIMING_LIB=<path>.
#   scripts/build_variants.sh timing "NAME:[extra nvcc flags]" ...   -> build/timing/t_NAME.so
# Every library is the full four-unit build (qpth_b200/build.py): the flags reach all units.
set -e
cd "$(dirname "$0")/.."
if [ "$1" != timing ]; then echo "usage: $0 timing NAME:[flags] ..." >&2; exit 2; fi
shift
dir=build/timing
mkdir -p $dir
for spec in "$@"; do
  name=${spec%%:*}; flags=${spec#*:}
  ( python -c "import sys; from qpth_b200 import build; build.build(force=True, extra=sys.argv[2:], out=sys.argv[1])" $PWD/$dir/t_$name.so -DQPB_TIMING $flags 2>&1 | grep -E "error" || true; echo "built $dir/t_$name.so [$flags]" ) &
done
wait
