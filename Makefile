# Builds the C-ABI CUDA library in-tree (sm_90a only) and the CPU-side test binaries.
NVCC ?= nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
GEN := build/gen
NVFLAGS := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xcompiler -Wall -I $(GEN)
SRC := sm3det_b200/csrc
OBJ := build/obj
LIB := sm3det_b200/lib/libsm3det_b200.so
SRCS := common.cu gemm_tc.cu ffn_fused.cu norm.cu stencil.cu front.cu moe.cu reduce.cu act.cu lsk.cu neck.cu rpn_head.cu capi.cu
OBJS := $(SRCS:%.cu=$(OBJ)/%.o)

all: $(LIB)

# inline-PTX wgmma wrappers, one operand list per N (generated)
$(GEN)/wgmma.cuh: tools/gen_wgmma.py
	@mkdir -p $(GEN)
	python3 tools/gen_wgmma.py $@

$(OBJ)/%.o: $(SRC)/%.cu $(wildcard $(SRC)/*.cuh) $(SRC)/kernels.h include/sm3det_b200.h $(GEN)/wgmma.cuh
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(LIB): $(OBJS)
	@mkdir -p sm3det_b200/lib
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -lcudart

build/gemm_test: tests/cuda/gemm_test.cu $(SRC)/gemm_tc.cu $(SRC)/common.cu $(SRC)/gemm_tc.cuh $(GEN)/wgmma.cuh
	@mkdir -p build
	$(NVCC) $(ARCH) -O3 -std=c++17 -lineinfo -I $(SRC) -I $(GEN) tests/cuda/gemm_test.cu $(SRC)/gemm_tc.cu $(SRC)/common.cu -o $@

build/ffn_test: tests/cuda/ffn_test.cu $(SRC)/ffn_fused.cu $(SRC)/gemm_tc.cu $(SRC)/common.cu $(SRC)/gemm_tc.cuh $(SRC)/ffn_fused.cuh $(GEN)/wgmma.cuh
	@mkdir -p build
	$(NVCC) $(ARCH) -O3 -std=c++17 -lineinfo -I $(SRC) -I $(GEN) tests/cuda/ffn_test.cu $(SRC)/ffn_fused.cu $(SRC)/gemm_tc.cu $(SRC)/common.cu -o $@

build/mma_bench: tests/cuda/mma_bench.cu $(SRC)/gemm_tc.cuh $(SRC)/common.cu $(GEN)/wgmma.cuh
	@mkdir -p build
	$(NVCC) $(ARCH) -O3 -std=c++17 -lineinfo -I $(SRC) -I $(GEN) tests/cuda/mma_bench.cu $(SRC)/common.cu -o $@

clean:
	rm -rf build sm3det_b200/lib/*.so

.PHONY: all clean
