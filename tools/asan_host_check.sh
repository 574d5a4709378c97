#!/bin/bash
# Host-side memory check of the product library (CPU only): the host C sources are rebuilt with AddressSanitizer, linked
# with the already compiled kernel objects into a scratch copy of libaudioflux_b200.so, and the CPU test groups that drive
# the library (constructors, tables, plans, streaming bookkeeping, C-ABI) run against it.  Nothing in the tree is modified.
# usage: tools/asan_host_check.sh            (after `make -C audioflux_b200/csrc`)
set -e
ROOT=$(cd "$(dirname "$0")/.." && pwd)
TMP=$(mktemp -d /tmp/afb200_asan.XXXXXX)
ASAN=$(gcc -print-file-name=libasan.so)
for f in "$ROOT"/audioflux_b200/csrc/host/*.c; do
  gcc -std=gnu99 -O1 -g -fPIC -fsanitize=address -fno-omit-frame-pointer -ffp-contract=off -I/usr/local/cuda/include -c "$f" -o "$TMP/$(basename "$f" .c).o"
done
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -Xlinker -Bsymbolic -o "$TMP/libaudioflux_b200.so" \
  "$TMP"/*.o "$ROOT"/audioflux_b200/csrc/build/*.cu.o -lm -Xlinker -lasan
cd "$ROOT"
export AFB200_LIB_PATH="$TMP/libaudioflux_b200.so"
LD_PRELOAD="$ASAN" ASAN_OPTIONS=detect_leaks=0 python -c "import audioflux_b200.lib as L; print('library under test:', L.LIB_PATH)"
LD_PRELOAD="$ASAN" ASAN_OPTIONS=detect_leaks=0 \
  python -m pytest tests/test_capi.py tests/test_tables.py tests/test_next_rows_cpu.py tests/test_reassign_cpu.py tests/test_deconv_cpu.py \
    tests/test_ctor_fuzz.py -x -q -p no:cacheprovider
rm -rf "$TMP"
