# ehb200 — builds the CUDA library (sm_90a only) and the CPU oracle.
NVCC      ?= nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVCCFLAGS := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall,-Wno-unused-function --expt-relaxed-constexpr
CSRC      := embeddinghub_b200/csrc
OBJDIR    := build/obj
SRCS      := $(wildcard $(CSRC)/*.cu)
OBJS      := $(patsubst $(CSRC)/%.cu,$(OBJDIR)/%.o,$(SRCS))
LIB       := embeddinghub_b200/libehb200.so

all: $(LIB) oracle tests/cpp/ann_index_cases tests/cpp/concurrent_search tests/cpp/sharded_two_dev tests/cpp/rwlock_stress \
     tests/cpp/exchange_layout \
     tests/cpp/libbf16_probe.so tests/cpp/libi8_probe.so tests/cpp/ann_index_bf16 tests/cpp/ann_index_by_key

# test-only extern "C" wrappers around the K3 launchers of the shipped library (run by tests/test_gpu_bf16_gemm.py)
tests/cpp/libbf16_probe.so: tests/cpp/bf16_probe.cu $(CSRC)/kernels.h $(LIB)
	$(NVCC) $(ARCH) -O2 -std=c++17 --expt-relaxed-constexpr -Xcompiler -fPIC,-Wall -shared -I$(CSRC) $< \
	  -Lembeddinghub_b200 -lehb200 -Xlinker -rpath,'$$ORIGIN/../../embeddinghub_b200' -o $@

# test-only extern "C" wrapper around the int8 screen-copy conversion (run by tests/test_gpu_walk_screen_int8.py)
tests/cpp/libi8_probe.so: tests/cpp/i8_probe.cu $(CSRC)/kernels.h $(LIB)
	$(NVCC) $(ARCH) -O2 -std=c++17 --expt-relaxed-constexpr -Xcompiler -fPIC,-Wall -shared -I$(CSRC) $< \
	  -Lembeddinghub_b200 -lehb200 -Xlinker -rpath,'$$ORIGIN/../../embeddinghub_b200' -o $@

# the reference's ANNIndex unit-test cases against the C++ drop-in twin (run by tests/test_gpu_host.py)
tests/cpp/ann_index_cases: tests/cpp/ann_index_cases.cc include/ehb200_ann_index.hpp $(LIB)
	g++ -std=c++17 -O2 -Iinclude $< -Lembeddinghub_b200 -lehb200 -Wl,-rpath,'$$ORIGIN/../../embeddinghub_b200' -o $@

# the C++ twin with a bf16 graph search (run by tests/test_gpu_bf16_walk.py)
tests/cpp/ann_index_bf16: tests/cpp/ann_index_bf16.cc include/ehb200_ann_index.hpp $(LIB)
	g++ -std=c++17 -O2 -Iinclude $< -Lembeddinghub_b200 -lehb200 -Wl,-rpath,'$$ORIGIN/../../embeddinghub_b200' -o $@

# key mode through the C++ twin (run by tests/test_gpu_search_by_label.py)
tests/cpp/ann_index_by_key: tests/cpp/ann_index_by_key.cc include/ehb200_ann_index.hpp $(LIB)
	g++ -std=c++17 -O2 -Iinclude $< -Lembeddinghub_b200 -lehb200 -Wl,-rpath,'$$ORIGIN/../../embeddinghub_b200' -o $@

# 64 pthreads issuing Q=1 searches through the C ABI (the cgo goroutine pattern; run by tests/test_gpu_round2.py)
tests/cpp/concurrent_search: tests/cpp/concurrent_search.c include/ehb200.h $(LIB)
	gcc -std=c11 -O2 -D_POSIX_C_SOURCE=200809L -Iinclude $< -Lembeddinghub_b200 -lehb200 -lpthread -lm -Wl,-rpath,'$$ORIGIN/../../embeddinghub_b200' -o $@

# host-only stress test of the reader/writer lock (run by tests/test_abi_cpu.py; no GPU needed)
tests/cpp/rwlock_stress: tests/cpp/rwlock_stress.cu $(CSRC)/index_impl.h
	$(NVCC) $(ARCH) -O2 -std=c++17 --expt-relaxed-constexpr $< -o $@ -lpthread

# host-only check of the shard exchange's buffer layout (run by tests/test_exchange_layout_cpu.py; no GPU needed)
tests/cpp/exchange_layout: tests/cpp/exchange_layout.cu $(CSRC)/exchange_layout.cuh
	$(NVCC) $(ARCH) -O2 -std=c++17 --expt-relaxed-constexpr -Xcompiler -Wall $< -o $@

# n_dev = 2 through the C ABI (run by tests/test_gpu_round2.py)
tests/cpp/sharded_two_dev: tests/cpp/sharded_two_dev.c include/ehb200.h $(LIB)
	gcc -std=c11 -O2 -Iinclude $< -Lembeddinghub_b200 -lehb200 -lm -Wl,-rpath,'$$ORIGIN/../../embeddinghub_b200' -o $@

$(OBJDIR)/%.o: $(CSRC)/%.cu $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) include/ehb200.h
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVCCFLAGS) -c $< -o $@

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS)

oracle:
	$(MAKE) -s -C oracle

clean:
	rm -rf build $(LIB)
	$(MAKE) -s -C oracle clean

.PHONY: all oracle clean
