# Builds the product library  vkfft_b200/lib/libb200fft.so  (CUDA, sm_90a only).
# `make -j8`; __graft_entry__.build() calls this.  Objects go to build/ (git-ignored).
NVCC      ?= nvcc
CXX       ?= g++
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := -std=c++17 -O3 $(ARCH) -lineinfo -Xcompiler -fPIC -Ivkfft_b200/csrc -Iinclude
CXXFLAGS  := -std=c++17 -O2 -fPIC -Ivkfft_b200/csrc -Iinclude
SRC       := vkfft_b200/csrc
SHARDS    := 0 1 2 3 4 5 6 7 8 9 10 11 12 13 14 15 16 17 18 19 20 21 22 23 24 25 26 27
SHARD_OBJ := $(foreach s,$(SHARDS),build/kernels_shard_$(s).o)
HDRS      := $(wildcard $(SRC)/*.cuh $(SRC)/*.h $(SRC)/*.def include/*.h)
LIB       := vkfft_b200/lib/libb200fft.so

all: $(LIB)

build/kernels_shard_%.o: $(SRC)/kernels_shard.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -DB2_SHARD=$* -c $< -o $@

build/kernels_generic.o: $(SRC)/kernels_generic.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -c $< -o $@

build/runtime.o: $(SRC)/runtime.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -c $< -o $@

build/window.o: $(SRC)/window.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -c $< -o $@

build/jit_headers.cpp: tools/embed_headers.py $(HDRS)
	@mkdir -p build
	python3 tools/embed_headers.py $@

build/jit_headers.o: build/jit_headers.cpp
	$(CXX) $(CXXFLAGS) -c $< -o $@

build/%.o: $(SRC)/%.cpp $(HDRS)
	@mkdir -p build
	$(CXX) $(CXXFLAGS) -c $< -o $@

$(LIB): $(SHARD_OBJ) build/kernels_generic.o build/runtime.o build/window.o build/planner.o build/kernel_registry.o build/jit.o build/jit_headers.o
	@mkdir -p vkfft_b200/lib
	$(NVCC) -shared $(ARCH) -o $@ $^ -lcudart_static -ldl -lrt -lpthread

clean:
	rm -rf build vkfft_b200/lib

.PHONY: all clean
