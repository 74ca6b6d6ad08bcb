#!/bin/bash
# usage: tools/build_variant.sh <name> [extra nvcc -D flags...]   -> nvdiffrecmc_b200/lib/variants/<name>.so
#        SRC=<dir> tools/build_variant.sh ...  compiles the sources of another directory (e.g. an older revision checked out to /tmp) --
#        the include path still points at this tree's include/mcshade.h, so the variant must have the same C ABI.
# The source list is the in-tree build's (nvdiffrecmc_b200/_lib.py SOURCES), so a variant exports every symbol _lib.lib() binds.
set -e
root="$(cd "$(dirname "$0")/.." && pwd)"
src="${SRC:-$root/nvdiffrecmc_b200/csrc}"
name=$1; shift
sources=$(cd "$root" && python3 -c "from nvdiffrecmc_b200._lib import SOURCES; print(*SOURCES)")
out="$root/nvdiffrecmc_b200/lib/variants"
mkdir -p "$out/obj_$name"
cd "$src"
for f in $sources; do
  nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC "$@" -c "$f" -o "$out/obj_$name/${f%.cu}.o" &
done
wait
nvcc -shared -gencode arch=compute_90a,code=sm_90a -o "$out/$name.so" "$out"/obj_$name/*.o
rm -rf "$out/obj_$name"
echo built $name
