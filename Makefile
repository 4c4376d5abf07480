# Builds libb2f.so (hand-written sm_90a kernels + C ABI) in-tree.
NVCC      ?= /usr/local/cuda/bin/nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xcompiler -Wall -cudart shared \
             --expt-relaxed-constexpr -Xptxas -v
CSRC      := gpt_image_edit_b200/csrc
LIBDIR    := gpt_image_edit_b200/lib
SRCS      := $(wildcard $(CSRC)/*.cu)
OBJS      := $(patsubst $(CSRC)/%.cu,build/%.o,$(SRCS))
HDRS      := $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) include/b2f.h
# only the b2f_* functions of include/b2f.h are exported
VERSION_SCRIPT := $(CSRC)/libb2f.map

all: $(LIBDIR)/libb2f.so

build/%.o: $(CSRC)/%.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> build/$*.ptxas.log || (cat build/$*.ptxas.log; exit 1)
	@grep -E "error|warning|spill|registers" build/$*.ptxas.log | grep -v "0 bytes spill" | head -40 || true

$(LIBDIR)/libb2f.so: $(OBJS) $(VERSION_SCRIPT)
	@mkdir -p $(LIBDIR)
	$(NVCC) $(ARCH) -shared -cudart shared -o $@ $(OBJS) -Xlinker -rpath -Xlinker /usr/local/cuda/lib64 \
		-Xlinker --version-script=$(VERSION_SCRIPT)

clean:
	rm -rf build $(LIBDIR)/libb2f.so

.PHONY: all clean
