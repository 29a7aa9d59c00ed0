#!/bin/bash
# Compile oracle/make_golden_checkpoint.cpp against the LibTorch bundled with the installed torch wheel and run it:
# -> tests/golden/libtorch_states.pt, tests/golden/libtorch_scalars.pt (the checkpoint-reader fixtures).
# usage: oracle/make_golden_checkpoint.sh            (from anywhere; about 15 s of g++)
set -eu
cd "$(dirname "$0")/.."
PY=${PY:-python}
TORCH=$($PY -c "import torch, os; print(os.path.dirname(torch.__file__))")
ABI=$($PY -c "import torch; print(int(torch._C._GLIBCXX_USE_CXX11_ABI))")
TMP=$(mktemp -d)
trap 'rm -rf "$TMP"' EXIT
g++ -std=c++17 -O1 -D_GLIBCXX_USE_CXX11_ABI=$ABI -I"$TORCH/include" -I"$TORCH/include/torch/csrc/api/include" \
    oracle/make_golden_checkpoint.cpp -o "$TMP/make_golden_checkpoint" \
    -L"$TORCH/lib" -Wl,--no-as-needed -ltorch -ltorch_cpu -lc10 -Wl,--as-needed -Wl,-rpath,"$TORCH/lib"
"$TMP/make_golden_checkpoint" tests/golden
ls -l tests/golden/libtorch_states.pt tests/golden/libtorch_scalars.pt
