# hpc-patterns-b200 — native build (sm_90a only).
#
#   make            everything: static lib, CLIs in bin/, torch extension (_C.so)
#   make cli        native CLIs only            make ext   torch extension only
#   make omp_con    host-only concurrency bench (plain g++ -fopenmp, no CUDA)
#   make sass       trimmed SASS listings + mnemonic summary -> docs/sass/
#   make sanitize   compute-sanitizer over the single-GPU kernel tests (needs a GPU)
#   make test       CPU test-suite (pytest -m "not gpu")
#
# Capability parity with the reference's build files: concurency/run_sycl.sh:6,
# run_omp.sh:6-7, p2p/run.sh:3-5, aurora.mpich.miniapps/src/CMakeLists.txt.
NVCC      ?= nvcc
# The image exports CXX=/opt/gcc/bin/g++, a wrapper that cannot link -fopenmp;
# always use the system compiler (override with HOSTCXX=...).
HOSTCXX   ?= $(shell command -v /usr/bin/g++ || echo g++)
override CXX := $(HOSTCXX)
PYTHON    ?= python
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := -ccbin $(HOSTCXX) $(ARCH) -lineinfo -O3 -std=c++17 -Xcompiler -fPIC,-fopenmp,-Wall -Icsrc
CXXFLAGS  := -O2 -std=c++17 -fPIC -fopenmp -Wall -Wextra -Icsrc -I/usr/local/cuda/include
BUILD     := build

KERNEL_SRC := $(wildcard csrc/kernels/*.cu)
COMMON_CPP := csrc/common/driver_api.cpp csrc/common/peer_mem.cpp csrc/p2p/topology_core.cpp
CON_CPP    := csrc/concurency/driver.cpp csrc/concurency/backend_cpu.cpp
LIB_OBJS   := $(KERNEL_SRC:csrc/%.cu=$(BUILD)/%.o) $(COMMON_CPP:csrc/%.cpp=$(BUILD)/%.o) \
              $(CON_CPP:csrc/%.cpp=$(BUILD)/%.o) $(BUILD)/concurency/backend_cuda.o
LIB        := $(BUILD)/libhpcp.a

# Programs built straight from one source file depend on every header (cheap and never stale).
HEADERS := $(shell find csrc -name '*.h' -o -name '*.hpp' -o -name '*.cuh')

CLIS := bin/concurency bin/omp_con bin/peer2pear bin/topology bin/allreduce bin/alltoall bin/halo bin/interop_torchless \
        bin/interop_driver bin/native_selftest

.PHONY: all cli aliases ext omp_con sass sanitize test clean
all: cli ext
cli: $(CLIS) aliases

# Program names of the reference as links to the programs here; defaults follow the name (see each main()):
#   <app>.<type> typed miniapps (CMakeLists.txt upstream), the three allreduce variants (allocation kind),
#   reduce_scatter / allgather (the reduce-scatter of the allreduce miniapp, the all-gather of the alltoall miniapp),
#   peer2pear_i / peer2pear_w (Isend/Irecv vs -DUSE_WIN builds, p2p/run.sh:4-5), sycl_con (run_sycl.sh:6),
#   omp_host_threads / omp_nowait (one build per mode upstream, run_omp.sh:6-7; the mode is argv[1] here).
aliases: $(CLIS)
	@for n in allreduce.float allreduce.int allreduce.double allreduce.long allreduce.short allreduce.uint allreduce.uchar \
	          allreduce.bfloat16 allreduce.half \
	          allreduce.float_int allreduce.double_int allreduce.long_int allreduce.2int allreduce.short_int \
	          allreduce-mpi-sycl.float allreduce-mpi-sycl.int \
	          allreduce-usm-mpi-omp-offload.float allreduce-map-mpi-omp-offload.float; do ln -sf allreduce bin/$$n; done
	@for n in halo.float halo.double halo.bfloat16 halo.half; do ln -sf halo bin/$$n; done
	@ln -sf allreduce bin/reduce_scatter; ln -sf alltoall bin/allgather
	@ln -sf peer2pear bin/peer2pear_i; ln -sf peer2pear bin/peer2pear_w
	@ln -sf concurency bin/sycl_con; ln -sf omp_con bin/omp_host_threads; ln -sf omp_con bin/omp_nowait

# -MMD: every object records the headers it includes (build/**/*.d), so editing a header rebuilds its users.
$(BUILD)/%.o: csrc/%.cu
	@mkdir -p $(dir $@)
	$(NVCC) $(NVFLAGS) -MMD -MF $(@:.o=.d) -c $< -o $@

$(BUILD)/%.o: csrc/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -MMD -MP -c $< -o $@

-include $(LIB_OBJS:.o=.d)

$(LIB): $(LIB_OBJS)
	ar rcs $@ $^

bin/concurency: csrc/concurency/main.cpp $(LIB) $(HEADERS)
	@mkdir -p bin
	$(NVCC) $(NVFLAGS) $< $(LIB) -o $@ -lgomp

omp_con: bin/omp_con
bin/omp_con: csrc/concurency/main.cpp csrc/concurency/driver.cpp csrc/concurency/backend_cpu.cpp \
             csrc/concurency/backend_nocuda.cpp $(HEADERS)
	@mkdir -p bin
	$(CXX) -O2 -std=c++17 -fopenmp -Wall -Wextra $(filter %.cpp,$^) -o $@

bin/peer2pear: csrc/p2p/peer2pear.cu $(LIB) $(HEADERS)
	@mkdir -p bin
	$(NVCC) $(NVFLAGS) $< $(LIB) -o $@ -lgomp

bin/topology: csrc/p2p/topology.cpp csrc/p2p/topology_core.cpp $(HEADERS)
	@mkdir -p bin
	$(CXX) $(CXXFLAGS) -DHPCP_TOPOLOGY_WITH_CUDA $(filter %.cpp,$^) -o $@ -L/usr/local/cuda/lib64 -lcudart_static -ldl -lrt -lpthread

bin/allreduce: csrc/miniapps/allreduce.cu $(LIB) $(HEADERS)
	@mkdir -p bin
	$(NVCC) $(NVFLAGS) $< $(LIB) -o $@ -lgomp

bin/alltoall: csrc/miniapps/alltoall.cu $(LIB) $(HEADERS)
	@mkdir -p bin
	$(NVCC) $(NVFLAGS) $< $(LIB) -o $@ -lgomp

bin/halo: csrc/miniapps/halo.cu $(LIB) $(HEADERS)
	@mkdir -p bin
	$(NVCC) $(NVFLAGS) $< $(LIB) -o $@ -lgomp

bin/interop_torchless: csrc/interop/interop_runtime_streams.cu $(LIB) $(HEADERS)
	@mkdir -p bin
	$(NVCC) $(NVFLAGS) $< $(LIB) -o $@ -lgomp

bin/interop_driver: csrc/interop/interop_driver_runtime.cu $(LIB) $(HEADERS)
	@mkdir -p bin
	$(NVCC) $(NVFLAGS) $< $(LIB) -o $@ -lgomp

# host-only unit tests of the native runtime (no GPU needed to run)
bin/native_selftest: csrc/tests/native_selftest.cpp csrc/concurency/driver.cpp csrc/p2p/topology_core.cpp $(HEADERS)
	@mkdir -p bin
	$(CXX) $(CXXFLAGS) csrc/tests/native_selftest.cpp csrc/concurency/driver.cpp csrc/p2p/topology_core.cpp \
	    -o $@ -L/usr/local/cuda/lib64 -lcudart_static -ldl -lrt -lpthread

ext: $(LIB)
	$(PYTHON) -m hpc_patterns_b200._build

sass: $(LIB)
	./scripts/make_sass.sh

# compute-sanitizer memcheck / racecheck / synccheck over the single-GPU kernel tests (GPU box)
sanitize: all
	./scripts/sanitize.sh

test:
	$(PYTHON) -m pytest tests -x -q -m "not gpu"

clean:
	rm -rf $(BUILD) bin hpc_patterns_b200/_C*.so
