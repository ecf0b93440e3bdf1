#!/bin/bash
# Development aid: run the CPU-side host tests with the C++ host mirror built under AddressSanitizer + UBSan.
# (The in-tree library is restored by rebuilding afterwards.)
set -e
cd "$(dirname "$0")/.."
g++ -std=c++17 -O1 -g -fsanitize=address,undefined -fno-omit-frame-pointer -fPIC -shared -Wall -Wno-sign-compare \
  -o delly_b200/libdelly_b200_host.so delly_b200/host/capi.cpp -Ldelly_b200 -l:libdelly_b200.so -Wl,-rpath,'$ORIGIN'
# the CPU-only stand-in of the tests (tests/standin/host_standin.cpp) under the same sanitizers: built here, newer than its sources, so the
# test fixture takes it as it is; removed afterwards so the next plain run rebuilds it
mkdir -p tests/standin/_build
g++ -std=c++17 -O1 -g -fsanitize=address,undefined -fno-omit-frame-pointer -fPIC -shared -w -Wl,-Bsymbolic -o tests/standin/_build/libhost_standin.so \
  tests/standin/host_standin.cpp -Loracle/_ref -l:libdelly_ref.so -Ldelly_b200 -l:libdelly_b200.so -Wl,-rpath,"$PWD/oracle/_ref" -Wl,-rpath,"$PWD/delly_b200"
LD_PRELOAD="$(gcc -print-file-name=libasan.so) $(gcc -print-file-name=libubsan.so)" ASAN_OPTIONS=detect_leaks=0:protect_shadow_gap=0 \
  python -m pytest tests/test_host_cluster.py tests/test_host_genotype.py tests/test_host_split.py tests/test_svanno.py tests/test_methyl.py tests/test_lr_full_chain.py tests/test_genotype_mode.py tests/test_multi_sample.py tests/test_seq_identity.py tests/test_svtset.py tests/test_edlib_compat.py tests/test_example_data.py \
  tests/test_sharded.py tests/test_contig_shard.py tests/test_lr_contig_shard.py -x -q -m "not gpu" \
  -p no:cacheprovider || true
rm -f tests/standin/_build/libhost_standin.so
touch delly_b200/host/capi.cpp
./build.sh > /dev/null
