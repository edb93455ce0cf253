# Build of libsce.so (the C-ABI engine), the standalone GEMM self-test and the oracle's C pieces.
NVCC ?= nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xptxas -v
CSRC := sparse_coding_b200/csrc
LIB := sparse_coding_b200/libsce.so
# one object per family of entry points (make -j compiles them side by side)
LIB_OBJS := $(patsubst %,build/%.o,sce_abi sce_plan sce_eval sce_track sce_similarity sce_rowpass sce_correlation)

all: $(LIB)

$(LIB): $(LIB_OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(LIB_OBJS)

build/sce_%.o: $(CSRC)/sce_%.cu $(CSRC)/*.cuh $(CSRC)/sce_tmap.h include/sce.h
	mkdir -p build
	$(NVCC) $(NVFLAGS) -c -o $@ $<

selftest: build/gemm_selftest build/gemm_cluster_selftest build/gemm_tall_selftest
build/gemm_selftest: tests/csrc/gemm_selftest.cu $(CSRC)/*.cuh $(CSRC)/sce_tmap.h
	mkdir -p build
	$(NVCC) $(NVFLAGS) -o $@ tests/csrc/gemm_selftest.cu

build/gemm_cluster_selftest: tests/csrc/gemm_cluster_selftest.cu $(CSRC)/*.cuh $(CSRC)/sce_tmap.h
	mkdir -p build
	$(NVCC) $(NVFLAGS) -o $@ tests/csrc/gemm_cluster_selftest.cu

build/gemm_tall_selftest: tests/csrc/gemm_tall_selftest.cu $(CSRC)/*.cuh $(CSRC)/sce_tmap.h
	mkdir -p build
	$(NVCC) $(NVFLAGS) -o $@ tests/csrc/gemm_tall_selftest.cu

probe: build/gemm_overlap_probe
build/gemm_overlap_probe: tools/gemm_overlap_probe.cu $(CSRC)/*.cuh $(CSRC)/sce_tmap.h
	mkdir -p build
	$(NVCC) $(NVFLAGS) -o $@ tools/gemm_overlap_probe.cu

clean:
	rm -f $(LIB) $(LIB_OBJS) build/gemm_selftest build/gemm_cluster_selftest build/gemm_tall_selftest build/gemm_overlap_probe
