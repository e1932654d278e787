# Build everything in-tree (the .so files travel to the GPU box with the snapshot; they are git-ignored).
#   make            -> product library, host library, oracle
#   make product    -> deep-prove_b200/libdeepprove_b200.so      (CUDA kernels + C ABI, sm_90a only)
#   make oracle     -> oracle/libdp_oracle.so                     (CPU restatement: TEST INFRASTRUCTURE)
#                      tests/libdp_oracle_model_io.so             (its model IO: output, verifier on a given output)
NVCC      ?= /usr/local/cuda/bin/nvcc
CXX       ?= g++
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -Wall -Xptxas -v
PKG       := deep-prove_b200
CSRC      := $(PKG)/csrc
CU_SRCS   := $(wildcard $(CSRC)/*.cu)
CU_OBJS   := $(patsubst $(CSRC)/%.cu,build/%.o,$(CU_SRCS))
CU_HDRS   := $(wildcard $(CSRC)/*.cuh) include/deepprove_b200.h include/dp_poseidon2_constants.h include/dp_blake3.h
HOST_SRCS := $(wildcard $(PKG)/host/*.cpp)
HOST_HDRS := $(wildcard $(PKG)/host/*.hpp) include/deepprove_b200.h include/dp_blake3.h
ORC_SRCS  := $(wildcard oracle/*.cpp)
ORC_HDRS  := $(wildcard oracle/*.hpp) include/dp_poseidon2_constants.h include/dp_blake3.h

all: product host oracle tools

product: $(PKG)/libdeepprove_b200.so
host: $(PKG)/libdeepprove_host.so
oracle: oracle/libdp_oracle.so tests/libdp_oracle_model_io.so tests/libdp_stream_queue_io.so

build/%.o: $(CSRC)/%.cu $(CU_HDRS)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> build/$*.ptxas.log || (cat build/$*.ptxas.log; exit 1)

$(PKG)/libdeepprove_b200.so: $(CU_OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(CU_OBJS)

$(PKG)/libdeepprove_host.so: $(HOST_SRCS) $(HOST_HDRS) $(PKG)/libdeepprove_b200.so
	$(CXX) -O2 -std=c++17 -fPIC -shared -Wall -Iinclude -o $@ $(HOST_SRCS) -L$(PKG) -ldeepprove_b200 -Wl,-rpath,'$$ORIGIN' -lpthread

oracle/libdp_oracle.so: $(ORC_SRCS) $(ORC_HDRS)
	$(CXX) -O3 -march=x86-64-v3 -std=c++17 -fPIC -shared -Wall -o $@ $(ORC_SRCS) -lpthread

tests/libdp_oracle_model_io.so: tests/oracle_model_io.cpp $(ORC_HDRS)
	$(CXX) -O3 -march=x86-64-v3 -std=c++17 -fPIC -shared -Wall -o $@ tests/oracle_model_io.cpp -lpthread

# the proof stream's queue under a fake job (tests/test_prove_stream_abi.py): no device needed
tests/libdp_stream_queue_io.so: tests/stream_queue_io.cpp $(PKG)/host/proof_queue.hpp include/deepprove_b200.h
	$(CXX) -O2 -std=c++17 -fPIC -shared -Wall -o $@ tests/stream_queue_io.cpp -lpthread

# device-vs-host self test of the field primitives and Poseidon2 (run by tests/test_gpu_baseline_size.py on the GPU box)
tools: $(PKG)/gl_selftest_bin
$(PKG)/gl_selftest_bin: tools/gl_selftest.cu $(CU_HDRS) $(HOST_HDRS)
	$(NVCC) $(ARCH) -O2 -std=c++17 -Iinclude -o $@ tools/gl_selftest.cu

# developer tools (not part of `all`): kernel micro-benchmarks and the CUPTI timeline / API-census library (tools/trace_*.py)
devtools: $(PKG)/kbench_bin $(PKG)/libdp_trace.so
$(PKG)/kbench_bin: tools/kbench.cu $(CU_HDRS)
	$(NVCC) $(ARCH) -O3 -std=c++17 -lineinfo -Iinclude -Xcompiler -pthread -o $@ tools/kbench.cu
$(PKG)/libdp_trace.so: tools/cupti_trace.cpp
	$(CXX) -O2 -shared -fPIC -I/usr/local/cuda/include -I/usr/local/cuda/extras/CUPTI/include -o $@ tools/cupti_trace.cpp -L/usr/local/cuda/lib64 -L/usr/local/cuda/extras/CUPTI/lib64 -lcupti -lcudart -Wl,-rpath,/usr/local/cuda/lib64

clean:
	rm -rf build $(PKG)/*.so oracle/*.so tests/*.so $(PKG)/gl_selftest_bin

.PHONY: all product host oracle tools devtools clean
