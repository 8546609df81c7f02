#!/bin/bash
# A/B build of libb200search.so with extra nvcc flags (or none: the sources as they stand), next to the default build:
#   tools/build_variant.sh ptxas_o1 "-Xptxas -O1"   ->  build_variants/libb200search_ptxas_o1.so
# Use with B200_LIB_PATH=build_variants/libb200search_<name>.so python bench.py --headline-only
set -e
name=$1; extra=$2
root=$(cd "$(dirname "$0")/.." && pwd)
tmp=$(mktemp -d)
mkdir -p "$tmp/myscaledb_b200" "$tmp/include" "$root/build_variants"
cp -r "$root/myscaledb_b200/csrc" "$tmp/myscaledb_b200/csrc"
cp "$root/include/b200_search.h" "$tmp/include/"
rm -f "$tmp"/myscaledb_b200/csrc/*.o
make -C "$tmp/myscaledb_b200/csrc" -j8 EXTRA="$extra" OUT="$root/build_variants/libb200search_$name.so" > /dev/null
rm -rf "$tmp"
echo "built build_variants/libb200search_$name.so"
