# Builds the product library (CUDA, sm_90a only) and the CPU oracle (test infrastructure).
NVCC ?= nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC -Xcompiler -fvisibility=hidden
CSRC := nerf_rpn_b200/csrc
OBJ := build/nms.o build/rpn_post.o build/conv3d_igemm.o build/conv3d_slab.o build/conv3d_wgrad.o build/pointwise.o build/groupnorm.o build/fcos_post.o build/swin.o build/eval.o build/targets.o build/train.o build/fcos_loss.o
LIB := nerf_rpn_b200/lib/libnerf_rpn_b200.so

all: $(LIB) oracle

$(LIB): $(OBJ) Makefile
	@mkdir -p $(dir $@)
	$(NVCC) -shared $(ARCH) -o $@ $(OBJ)

build/%.o: $(CSRC)/%.cu $(wildcard $(CSRC)/*.cuh) include/nerf_rpn_b200.h Makefile
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -c $< -o $@

oracle:
	$(MAKE) -s -C oracle

clean:
	rm -rf build $(LIB) oracle/libbox_oracle.so

.PHONY: all oracle clean
