#!/bin/bash
# Is the DEVICE code of the working tree byte-identical to a given commit's?  (Used when host code changes without a GPU at hand: the GPU
# test results of <commit> then still describe the device code of the working tree.)   usage: profiles/sass_identity.sh <commit>
set -eu
ref=${1:?commit}
root=$(cd "$(dirname "$0")/.." && pwd)
tmp=$(mktemp -d)
trap 'rm -rf "$tmp"' EXIT
git -C "$root" archive "$ref" vulkan-path-tracer_b200 include | tar -x -C "$tmp"
(cd "$tmp/vulkan-path-tracer_b200" && make -j8 >/dev/null 2>&1)
(cd "$root/vulkan-path-tracer_b200" && make -j8 >/dev/null 2>&1)
# the tag nvcc gives an anonymous namespace (_GLOBAL__N__<hash>_) depends on the build directory, so it is left out
sig() { for f in "$1"/build/*.o; do echo "$(basename "$f") $(cuobjdump -sass "$f" 2>/dev/null | grep -v '^Fatbin\|^====\|arch =\|code version\|host =\|compile_size\|identifier' | sed 's/_GLOBAL__N__[0-9a-f]*_/_GLOBAL__N__/g' | md5sum | cut -c1-16)"; done; }
if diff <(sig "$tmp/vulkan-path-tracer_b200") <(sig "$root/vulkan-path-tracer_b200"); then echo "device SASS identical to $ref"; else echo "device SASS DIFFERS from $ref"; exit 1; fi
