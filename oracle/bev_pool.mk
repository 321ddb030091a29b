# oracle/bev_pool.mk — TEST-ONLY checkers for BEVPoolV2 (driven by oracle/bev_pool.py:build()). Nothing built here is
# linked into the product library.
#
#   make -f bev_pool.mk oracle : _build/libbev_pool_oracle.so — bev_pool_cpu.c (gcc)
#   make -f bev_pool.mk ref    : _ref/libref_bev_pool.so — the reference's BEVPoolV2 kernel translation units compiled
#                                UNMODIFIED from where they lie under $(REFERENCE), plus ref_bev_pool_shim.cu (ours),
#                                which only exports their launchers as extern "C". Skipped when $(REFERENCE) is absent.
REFERENCE ?= /root/reference
NVCC      ?= /usr/local/cuda/bin/nvcc
CC        ?= gcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
R         := $(REFERENCE)/TensorRT

oracle: _build/libbev_pool_oracle.so

_build/libbev_pool_oracle.so: bev_pool_cpu.c
	@mkdir -p _build
	$(CC) -O2 -ffp-contract=off -fno-fast-math -fPIC -shared -o $@ bev_pool_cpu.c -lm

REF_TUS := $(R)/plugin/bev_pool_v2/bevPoolKernel.cu \
           $(REFERENCE)/third_party/bev_mmdet3d/ops/bev_pool_v2/src/bev_pool_cuda.cu
REF_INC := -I stub -I $(R)/common -I $(R)/plugin/bev_pool_v2

ref:
	@if [ -d "$(REFERENCE)/TensorRT" ]; then $(MAKE) -f bev_pool.mk _ref/libref_bev_pool.so; \
	 else echo "oracle: $(REFERENCE) absent - keeping prebuilt oracle/_ref"; fi

_ref/libref_bev_pool.so: ref_bev_pool_shim.cu
	@mkdir -p _ref
	$(NVCC) $(ARCH) -std=c++17 -O3 -Xcompiler -fPIC -shared $(REF_INC) -o $@ ref_bev_pool_shim.cu $(REF_TUS)

.PHONY: oracle ref
