#!/usr/bin/env bash
# Builds libea_b200.so (sm_90a, H100) in-tree next to the sources' package: easyanimate_b200/libea_b200.so
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="$HERE/../libea_b200.so"
OBJ="$HERE/../_build"
mkdir -p "$OBJ"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
ARCH=(-gencode arch=compute_90a,code=sm_90a)
FLAGS=("${ARCH[@]}" -O3 -std=c++17 -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr -Xptxas -v -I"$HERE/../../include")
# objects of an earlier build for another architecture are rebuilt
if [[ ! -f "$OBJ/.arch" || "$(cat "$OBJ/.arch")" != "${ARCH[*]}" ]]; then rm -f "$OBJ"/*.o; echo "${ARCH[*]}" > "$OBJ/.arch"; fi
# an object is stale when it is older than its source or than any header a source can include
headers=("$HERE"/*.cuh "$HERE"/*.h "$HERE/../../include/ea_b200.h")
stale() {
  local dep
  for dep in "$@"; do [[ "$dep" -nt "$obj" ]] && return 0; done
  return 1
}
pids=()
objs=()
for src in "$HERE"/*.cu; do
  obj="$OBJ/$(basename "${src%.cu}").o"
  objs+=("$obj")
  if [[ ! -f "$obj" ]] || stale "$src" "${headers[@]}"; then
    ( "$NVCC" "${FLAGS[@]}" -c "$src" -o "$obj" > "$obj.log" 2>&1 || { cat "$obj.log"; exit 1; } ) &
    pids+=($!)
  fi
done
for p in "${pids[@]:-}"; do [[ -n "$p" ]] && wait "$p"; done
"$NVCC" "${ARCH[@]}" -shared -o "$OUT" "${objs[@]}" -lcudart_static -ldl -lrt -lpthread
echo "built $OUT"
