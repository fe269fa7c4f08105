#!/bin/bash
# A/B builds of librxb200.so: the same sources with different -D switches of fm_kernels.cu, one .so per variant
# under rx_tools_b200/variants/ (git-ignored; selected with RXB200_LIB=...).
#   tools/build_variants.sh name1="-DX=1 -DY=2" name2="..."
set -e
cd "$(dirname "$0")/../rx_tools_b200/csrc"
make -s -j4 >/dev/null            # every other object comes from the default build
others=$(make -s print-objs | tr ' ' '\n' | grep -vx fm_kernels.o)
ARCH="-gencode arch=compute_90a,code=sm_90a"
mkdir -p ../variants
pids=()
for spec in "$@"; do
	name="${spec%%=*}"; flags="${spec#*=}"
	(
		nvcc $ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xptxas -v $flags -c -o ../variants/fm_$name.o fm_kernels.cu 2> ../variants/fm_$name.ptxas.log
		nvcc $ARCH -shared -o ../variants/librxb200_$name.so ../variants/fm_$name.o $others -ldl
		echo "$flags" > ../variants/$name.flags
		echo "built $name: $flags"
	) &
	pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
