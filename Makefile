# Builds the sm_90a extension in-tree: sliders_b200/libsb200.so (C ABI declared in include/sb200.h).
# `python -c "import __graft_entry__ as g; g.build()"` runs the same recipe.
NVCC      ?= /usr/local/cuda/bin/nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVCCFLAGS := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xcompiler -Wall \
             --expt-relaxed-constexpr -Xptxas -v
CSRC      := sliders_b200/csrc
SRCS      := $(CSRC)/api.cu $(CSRC)/gemm.cu $(CSRC)/attention.cu $(CSRC)/norm.cu $(CSRC)/elementwise.cu $(CSRC)/attention_bwd.cu $(CSRC)/backward.cu
OBJS      := $(SRCS:.cu=.o)
LIB       := sliders_b200/libsb200.so

all: $(LIB)

$(CSRC)/%.o: $(CSRC)/%.cu $(CSRC)/common.h $(CSRC)/ptx.cuh $(CSRC)/wgmma.cuh include/sb200.h
	$(NVCC) $(NVCCFLAGS) -c $< -o $@ 2> $@.log || (cat $@.log; exit 1)
	@grep -E "registers|spill|error|warning" $@.log | sort | uniq -c | sort -rn | head -20 || true

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS)

clean:
	rm -f $(OBJS) $(CSRC)/*.o.log $(LIB)

.PHONY: all clean
