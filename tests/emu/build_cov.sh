#!/bin/sh
# Coverage build of the host emulation (tests only): the kernel sources compiled with --coverage, so that gcov can
# say which lines and branches of the kernels a test run reached.  Usage:
#   sh tests/emu/build_cov.sh /tmp/cov
#   WB_EMU_LIB=/tmp/cov/libworld_b200_emu_cov.so python -m pytest tests/test_emu_f0_tail.py -q
#   python tests/emu/cov_report.py /tmp/cov            # the F0 decision kernels; FILE:FUNCTION,... for others
# The counters (*.gcda) accumulate over runs in the output directory: remove them to start a new reading.
set -e
OUT=${1:-/tmp/cov}
cd "$(dirname "$0")"
SRC=$(cd ../../world_b200/csrc && pwd)   # absolute: gcov finds the sources from any directory
mkdir -p "$OUT"
for f in wb_api wb_rng wb_cheaptrick wb_d4c wb_stonemask wb_synthesis wb_codec wb_fileio wb_matlab wb_f0common wb_dio wb_harvest wb_host wb_multi; do
  g++ -x c++ -std=c++17 -O1 -g --coverage -fPIC -DWB_EMU -ffp-contract=off -mfma \
      -I../../include -c $SRC/$f.cu -o "$OUT/$f.o" &
done
wait
g++ -O1 -g -fPIC -DWB_EMU -c emu_globals.cpp -o "$OUT/emu_globals.o"
g++ -shared --coverage -o "$OUT/libworld_b200_emu_cov.so" "$OUT"/*.o -lm
echo "built $OUT/libworld_b200_emu_cov.so"
