#!/bin/bash
# A/B of the resident-CTAs-per-SM choice of the persistent line kernels (KL_B256 / KL_B320 / KL_B384, compile time):
# builds two more copies of the library outside the tree (no GPU needed), then times all three on a GPU.
#   tools/occ_ab.sh build      tools/occ_ab.sh run      (OCC_DIR: where the copies go, default /tmp/htv_occ)
set -e
cd "$(dirname "$0")/.."
C=hacktv_b200/csrc
D=${OCC_DIR:-/tmp/htv_occ}
if [ "$1" = build ]; then
	make -C $C > /dev/null
	mkdir -p $D
	NV="-O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -fmad=false -I include -I $C"
	nvcc $NV -DKL_B256=4 -DKL_B320=3 -DKL_B384=2 -c $C/htv_kernels.cu -o $D/hk_occ1.o
	nvcc $NV -DKL_B256=3 -DKL_B320=4 -DKL_B384=2 -c $C/htv_kernels.cu -o $D/hk_occ2.o
	for v in 1 2; do nvcc -shared -o $D/libhacktv_b200_occ$v.so $C/htv_tables.o $C/htv_modes.o $C/htv_host.o $C/htv_av_test.o $C/htv_rf.o $D/hk_occ$v.o -lm; done
	ls -la $D/*.so
else
	for lib in $PWD/hacktv_b200/libhacktv_b200.so $D/libhacktv_b200_occ1.so $D/libhacktv_b200_occ2.so; do
		echo "== $lib"
		HTV_LIB=$lib python tools/occ_time.py || true
	done
fi
