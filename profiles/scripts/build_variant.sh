#!/bin/bash
# A/B builds: build_variant.sh <name> <source.cu> "<-DFLAG=.. ...>"  ->  trajectoryoptimization.jl_b200/variants/lib_<name>.so
# (git-ignored); run with LIBTRAJOPT_B200=<path>.  One source file is recompiled with the flags, the rest is linked as built -- the objects
# of the integration rules other than RK4 (forward_r*.o, rollout_r*.o) included, so a variant of forward.cu or rollout.cu changes the RK4 kernels.
# VARIANT_DIR=<dir> puts the library and the variant object there instead (for a tree that cannot be written to).
set -e
name=$1; src=$2; flags=$3
cd "$(dirname "$0")/../../trajectoryoptimization.jl_b200/csrc"
make -s > /dev/null
out=${VARIANT_DIR:-../variants}; objdir=${VARIANT_DIR:-_build/variants}
mkdir -p $out $objdir
base=$(basename $src .cu)
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -ccbin /usr/bin/g++ -Xcompiler -fPIC -Xptxas -v $flags \
    -c $src -o $objdir/${base}_$name.o 2> $objdir/${base}_$name.log
objs=""
for o in capi rollout sweep riccati riccati_small lie riccati_frag forward solve; do
  if [ "$o" == "$base" ]; then objs="$objs $objdir/${base}_$name.o"; else objs="$objs _build/$o.o"; fi
done
objs="$objs $(ls _build/forward_r[0-9].o _build/rollout_r[0-9].o)"
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -ccbin /usr/bin/g++ -o $out/lib_$name.so $objs
echo "$name: $(grep -E 'Used|spill' $objdir/${base}_$name.log | sort | uniq -c | sort -rn | head -3 | tr '\n' ' ')"
