#!/usr/bin/env bash
# Builds the softmin probe pair (softmin_probe_pair.cu) against the engine's internal header, like plugins_example/build.sh.
# The library finds libmppi_b200.so relative to itself, so the tree can be moved after the build.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
CUDA_HOME="${CUDA_HOME:-/usr/local/cuda}"
"$CUDA_HOME/bin/nvcc" -std=c++17 -O3 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -shared \
  -o "$HERE/libmppi_plugin_softmin_probe.so" "$HERE/softmin_probe_pair.cu" -I"$HERE/../../include" \
  -L"$HERE/../../mppi-generic_b200" -Xlinker -rpath -Xlinker '$ORIGIN/../../mppi-generic_b200' -l:libmppi_b200.so \
  -L"$CUDA_HOME/lib64" -lcurand -lcufft
echo "built $HERE/libmppi_plugin_softmin_probe.so"
