# Builds the C-ABI CUDA library (sm_90a, H100) and the CPU oracle.
NVCC ?= nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := -O3 -std=c++17 $(ARCH) -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=hidden \
           --expt-relaxed-constexpr -Xptxas -v
CSRC := splatam_b200/csrc
OBJS := $(CSRC)/abi.o $(CSRC)/radix_sort.o $(CSRC)/project.o $(CSRC)/binning.o $(CSRC)/blend_forward.o \
        $(CSRC)/blend_backward.o $(CSRC)/geometry_backward.o $(CSRC)/train_ops.o $(CSRC)/prepare.o $(CSRC)/sh.o \
        $(CSRC)/map_ops.o $(CSRC)/eval_metrics.o $(CSRC)/ingest.o $(CSRC)/lpips.o \
        $(CSRC)/eval_frames.o
LIB := splatam_b200/libsplatam_b200.so

all: $(LIB) oracle

$(CSRC)/%.o: $(CSRC)/%.cu $(CSRC)/common.cuh $(CSRC)/pipeline.cuh $(CSRC)/radix_sort.cuh include/splatam_b200.h Makefile
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> $@.log || (cat $@.log; exit 1)

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -lcudart_static -Xcompiler -fvisibility=hidden

oracle:
	$(MAKE) -C oracle

clean:
	rm -f $(CSRC)/*.o $(CSRC)/*.o.log $(LIB)
	$(MAKE) -C oracle clean

.PHONY: all oracle clean
