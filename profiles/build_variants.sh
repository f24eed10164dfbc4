#!/bin/bash
# A/B builds of the Riccati kernel: build_variants.sh name "-DFLAG=.. -DFLAG=.." [name flags ...]
# -> trajectoryoptimization.jl_b200/variants/lib_<name>.so (git-ignored); run with LIBTRAJOPT_B200=<path>
set -e
cd "$(dirname "$0")/../trajectoryoptimization.jl_b200/csrc"
make -s > /dev/null
mkdir -p ../variants _build/variants
while [ $# -ge 2 ]; do
  name=$1; flags=$2; shift 2
  /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -ccbin /usr/bin/g++ -Xcompiler -fPIC -Xptxas -v $flags \
      -c riccati.cu -o _build/variants/riccati_$name.o 2> _build/variants/riccati_$name.log &
done
wait
for o in _build/variants/riccati_*.o; do
  name=$(basename $o .o); name=${name#riccati_}
  /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -ccbin /usr/bin/g++ -o ../variants/lib_$name.so _build/capi.o _build/rollout.o _build/sweep.o $o _build/riccati_small.o _build/lie.o _build/riccati_frag.o _build/forward.o _build/solve.o \
      _build/forward_r[0-9].o _build/rollout_r[0-9].o
  echo "$name: $(grep -A2 'k_riccatiILi13ELi4ELi2ELb1ELb1ELi' _build/variants/riccati_$name.log | grep -E 'Used|spill' | tr '\n' ' ')"
done
