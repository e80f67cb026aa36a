#!/bin/bash
# Build kernel variants of zb_kernels.cu (compile-time schedule parameters) as zlib_rs_b200/variants/libz_b200_<name>.so.
# usage: build_variants.sh name1:"-DZB_T_CMP=16" name2:"-DZB_T_CMP=16 -DZB_WALK_BURST=8" ...
set -e
cd "$(dirname "$0")/../zlib_rs_b200/csrc"
make -j8 > /dev/null
mkdir -p ../variants _build/var
ARCH="-gencode arch=compute_90a,code=sm_90a"
for spec in "$@"; do
  name=${spec%%:*}; flags=${spec#*:}
  ( nvcc $ARCH -std=c++17 -O3 -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -diag-suppress 177 -rdc=false $flags -c zb_kernels.cu -o _build/var/zb_kernels_$name.o && nvcc $ARCH -std=c++17 -O3 -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -diag-suppress 177 -rdc=false $flags -c zb_engine.cu -o _build/var/zb_engine_$name.o && nvcc $ARCH -std=c++17 -O3 -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -diag-suppress 177 -rdc=false $flags -c ${SLOW_SRC:-zb_slow.cu} -o _build/var/zb_slow_$name.o &&
    nvcc $ARCH -shared -o ../variants/libz_b200_$name.so _build/var/zb_kernels_$name.o _build/var/zb_slow_$name.o _build/zb_serial.o _build/zb_checksum.o _build/var/zb_engine_$name.o _build/zb_inflate.o _build/zb_zlib.o -lcudart_static -lpthread -ldl -lrt -Xlinker -Bsymbolic && echo "built $name ($flags)" ) &
done
wait
