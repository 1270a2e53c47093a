# Builds libparseable_b200.so (CUDA, sm_90a only) in-tree, the C oracle and the
# CPU test harness for the pure decode functions.  No PyTorch, no Triton.
NVCC      ?= /usr/local/cuda/bin/nvcc
CXX       ?= g++
CC        ?= gcc
PY_NCCL   := $(shell python -c "import nvidia.nccl,os;print(os.path.dirname(nvidia.nccl.__file__))" 2>/dev/null)
NCCL_INC  := $(if $(PY_NCCL),-I$(PY_NCCL)/include,)
# link the torch-bundled libnccl.so.2 when present (same soname as the system one, so a
# process that also imports torch ends up with a single NCCL)
NCCL_LIB  := $(if $(PY_NCCL),-L$(PY_NCCL)/lib -l:libnccl.so.2 -Xlinker -rpath -Xlinker $(PY_NCCL)/lib,-lnccl)
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall,-Wno-unused-function --expt-relaxed-constexpr $(NCCL_INC) -Iinclude $(EXTRA)
CSRC      := parseable_b200/csrc
OBJDIR    ?= build
LIB       ?= parseable_b200/libparseable_b200.so
EXTRA     ?=

CU_SRCS   := $(CSRC)/table.cu $(CSRC)/query.cu
CPP_SRCS  := $(CSRC)/parquet_meta.cpp $(CSRC)/arrow_export.cpp $(CSRC)/capi.cpp $(CSRC)/comm.cpp $(CSRC)/planning.cpp \
             $(CSRC)/regex_compile.cpp
OBJS      := $(patsubst $(CSRC)/%.cu,$(OBJDIR)/%.o,$(CU_SRCS)) $(patsubst $(CSRC)/%.cpp,$(OBJDIR)/%.o,$(CPP_SRCS))
HDRS      := $(wildcard $(CSRC)/*.hpp $(CSRC)/*.cuh $(CSRC)/*.inc include/*.h)
# the same library on a host-staged communicator (tools/comm_host.cpp, no NCCL): several ranks as processes on one
# device, for tests only (PQB_LIB selects it)
HOSTCOMM_LIB  := tools/libparseable_b200_hostcomm.so
HOSTCOMM_OBJS := $(filter-out $(OBJDIR)/comm.o,$(OBJS)) $(OBJDIR)/comm_host.o

all: $(LIB) $(HOSTCOMM_LIB) oracle tools

$(OBJDIR)/%.o: $(CSRC)/%.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> $(OBJDIR)/$*.ptxas.log || (cat $(OBJDIR)/$*.ptxas.log; false)

$(OBJDIR)/%.o: $(CSRC)/%.cpp $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -x cu -c $< -o $@

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -lcudart $(NCCL_LIB)

$(OBJDIR)/comm_host.o: tools/comm_host.cpp $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -I$(CSRC) -x cu -c $< -o $@
$(HOSTCOMM_LIB): $(HOSTCOMM_OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(HOSTCOMM_OBJS) -lcudart

oracle: oracle/liboracle.so
oracle/liboracle.so: oracle/oracle.c
	$(CC) -O2 -std=c11 -fPIC -shared -Wall -o $@ $< -lm

tools: tools/libdecode_core_host.so tools/libzstd_host.so tools/libjson_host.so tools/liborder_keys_host.so tools/libregex_host.so \
       tools/liblz_host.so tools/liblz_host_desc.so tools/libdecomp_dev.so tools/libhash_merge_host.so tools/libin_set_host.so
# the LZ4_RAW / SNAPPY decoders on the host, lanes in ascending and in descending order
tools/liblz_host.so: tools/lz_host.cpp $(CSRC)/lz_decode.cuh $(CSRC)/zstd_decode.cuh
	$(CXX) -O2 -std=c++17 -fPIC -shared -Wall -I$(CSRC) -o $@ $<
tools/liblz_host_desc.so: tools/lz_host.cpp $(CSRC)/lz_decode.cuh $(CSRC)/zstd_decode.cuh
	$(CXX) -O2 -std=c++17 -fPIC -shared -Wall -DLZ_LANES_DESCENDING=1 -I$(CSRC) -o $@ $<
# the page decoder kernels, launched as table.cu launches them (GPU tests only)
tools/libdecomp_dev.so: tools/decomp_dev.cu $(HDRS)
	$(NVCC) $(NVFLAGS) -I$(CSRC) -shared -o $@ $< -lcudart
tools/libregex_host.so: tools/regex_host.cpp $(CSRC)/regex_compile.cpp $(CSRC)/regex_compile.hpp $(CSRC)/regex_match.cuh $(CSRC)/regex_unicode.inc
	$(CXX) -O2 -std=c++17 -fPIC -shared -Wall -I$(CSRC) -o $@ $<
tools/liborder_keys_host.so: tools/order_keys_host.cpp $(CSRC)/order_keys.cuh $(CSRC)/percentile_core.cuh $(CSRC)/decode_core.cuh $(CSRC)/device_structs.hpp
	$(CXX) -O2 -std=c++17 -ffp-contract=off -fPIC -shared -Wall -I$(CSRC) -o $@ $<
# the merge of a hashed GROUP BY's rank tables on the host (f64 sums bit for bit: no contraction)
tools/libhash_merge_host.so: tools/hash_merge_host.cpp $(CSRC)/hash_merge.cuh $(CSRC)/decode_core.cuh $(CSRC)/device_structs.hpp
	$(CXX) -O2 -std=c++17 -ffp-contract=off -fPIC -shared -Wall -I$(CSRC) -o $@ $<
# the membership set of PQ_OP_IN on the host
tools/libin_set_host.so: tools/in_set_host.cpp $(CSRC)/in_set.cuh $(CSRC)/decode_core.cuh $(CSRC)/device_structs.hpp
	$(CXX) -O2 -std=c++17 -fPIC -shared -Wall -I$(CSRC) -o $@ $<
tools/libjson_host.so: tools/json_host.cpp $(CSRC)/json_egress.cuh $(CSRC)/ryu_f64.cuh $(CSRC)/ryu_tables.inc
	$(CXX) -O2 -std=c++17 -fPIC -shared -Wall -Wno-maybe-uninitialized -I$(CSRC) -o $@ $<
tools/libzstd_host.so: tools/zstd_host.cpp $(CSRC)/zstd_decode.cuh $(CSRC)/inflate_decode.cuh
	$(CXX) -O2 -std=c++17 -fPIC -shared -Wall -I$(CSRC) -o $@ $<
tools/libdecode_core_host.so: tools/decode_core_host.cpp $(CSRC)/decode_core.cuh $(CSRC)/device_structs.hpp
	$(CXX) -O2 -std=c++17 -fPIC -shared -Wall -I$(CSRC) -o $@ $<

clean:
	rm -rf $(OBJDIR) $(LIB) $(HOSTCOMM_LIB) oracle/liboracle.so tools/libdecode_core_host.so tools/libzstd_host.so tools/libjson_host.so tools/liborder_keys_host.so tools/libregex_host.so \
	      tools/liblz_host.so tools/liblz_host_desc.so tools/libdecomp_dev.so tools/libhash_merge_host.so tools/libin_set_host.so

.PHONY: all oracle tools clean
