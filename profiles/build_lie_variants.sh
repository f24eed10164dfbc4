#!/bin/bash
# A/B builds of lie.cu (tensor-core Riccati pass on the materialised expansion): build_lie_variants.sh name "-DFLAG=.." [name flags ...]
# -> trajectoryoptimization.jl_b200/variants/lib_lie_<name>.so (git-ignored); run with LIBTRAJOPT_B200=<path>
set -e
cd "$(dirname "$0")/../trajectoryoptimization.jl_b200/csrc"
make -s > /dev/null
mkdir -p ../variants _build/variants
while [ $# -ge 2 ]; do
  name=$1; flags=$2; shift 2
  /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -ccbin /usr/bin/g++ -Xcompiler -fPIC -Xptxas -v $flags \
      -c lie.cu -o _build/variants/lie_$name.o 2> _build/variants/lie_$name.log
  /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -ccbin /usr/bin/g++ -o ../variants/lib_lie_$name.so _build/capi.o _build/rollout.o _build/sweep.o _build/riccati.o _build/riccati_small.o _build/variants/lie_$name.o _build/riccati_frag.o _build/forward.o _build/solve.o _build/forward_r[0-9].o _build/rollout_r[0-9].o
  echo "$name: $(grep -A2 'k_riccati_dense_mmaILi[0-9]*ELb1E' _build/variants/lie_$name.log | grep -E 'Used|spill' | tr '\n' ' ')"
done
