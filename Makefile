# Builds libfi_epp.so (sm_90a CUDA + host C++) in-tree, and the CPU oracle.
NVCC ?= /usr/local/cuda/bin/nvcc
CXX ?= g++
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall,-Wextra,-Wno-unused-parameter -Xptxas -v
CSRC := fusioninfer_b200/csrc
OBJDIR := build
LIB := fusioninfer_b200/lib/libfi_epp.so
HOSTCHECK := fusioninfer_b200/lib/libfi_hostcheck.so

CU_SRCS := $(CSRC)/hash_kernels.cu $(CSRC)/index_kernels.cu $(CSRC)/lru_kernels.cu $(CSRC)/match_kernels.cu \
           $(CSRC)/engine.cu $(CSRC)/engine_index.cu $(CSRC)/engine_lru.cu $(CSRC)/engine_pick.cu \
           $(CSRC)/engine_snapshot.cu $(CSRC)/engine_comm.cu
CU_OBJS := $(patsubst $(CSRC)/%.cu,$(OBJDIR)/%.o,$(CU_SRCS))
HDRS := $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) include/fi_epp.h

EXT_ORACLE := $(OBJDIR)/libepp_ext_oracle.so
RESIZE_ORACLE := $(OBJDIR)/libepp_resize_oracle.so
SNAPSHOT_ORACLE := $(OBJDIR)/libepp_snapshot_oracle.so
COUNTS_ORACLE := $(OBJDIR)/libepp_counts_oracle.so

all: $(LIB) $(HOSTCHECK) oracle $(EXT_ORACLE) $(RESIZE_ORACLE) $(SNAPSHOT_ORACLE) $(COUNTS_ORACLE)

$(OBJDIR)/%.o: $(CSRC)/%.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> $(OBJDIR)/$*.ptxas.log || (cat $(OBJDIR)/$*.ptxas.log; false)

$(OBJDIR)/epp_config.o: $(CSRC)/epp_config.cpp include/fi_epp.h
	@mkdir -p $(OBJDIR)
	$(CXX) -O2 -std=c++17 -fPIC -Wall -Wextra -c $< -o $@

$(LIB): $(CU_OBJS) $(OBJDIR)/epp_config.o
	@mkdir -p $(dir $(LIB))
	$(NVCC) $(ARCH) -shared -o $@ $^ -ldl

# host-only build of the shared host/device arithmetic, for CPU unit tests
$(HOSTCHECK): $(CSRC)/hostcheck.cpp $(CSRC)/xxh64.cuh $(CSRC)/bitslice.cuh $(CSRC)/lru.h $(CSRC)/lru_batch.h $(CSRC)/lru_plan.h $(CSRC)/pool_shape.h $(CSRC)/snapshot_format.h $(CSRC)/tiebreak.cuh
	@mkdir -p $(dir $(HOSTCHECK))
	$(CXX) -O2 -std=c++17 -ffp-contract=off -fPIC -Wall -Wextra -shared -pthread -x c++ $(CSRC)/hostcheck.cpp -o $@

oracle:
	$(MAKE) -C oracle

# a test-side extension of the CPU oracle, tests/<name>.cpp -> build/libepp_<name>.so (test infrastructure only):
# tests/ext_oracle.cpp adds the ranked / subset pick and per-endpoint LRU capacities
$(OBJDIR)/libepp_%.so: tests/%.cpp oracle/epp_oracle.cpp include/fi_epp.h
	@mkdir -p $(OBJDIR)
	$(CXX) -O2 -std=c++17 -ffp-contract=off -fPIC -Wall -Wextra -pthread -shared -o $@ $<
# tests/resize_oracle.cpp adds the pool resize on top of tests/ext_oracle.cpp
$(RESIZE_ORACLE): tests/ext_oracle.cpp
# tests/snapshot_oracle.cpp adds the state of an index snapshot on top of tests/resize_oracle.cpp
$(SNAPSHOT_ORACLE): tests/ext_oracle.cpp tests/resize_oracle.cpp
# tests/counts_oracle.cpp adds the match counts of fi_epp_match_counts on top of tests/ext_oracle.cpp
$(COUNTS_ORACLE): tests/ext_oracle.cpp

clean:
	rm -rf $(OBJDIR) $(LIB) $(HOSTCHECK)
	$(MAKE) -C oracle clean

.PHONY: all oracle clean

# debug variant with per-phase clock64 sums inside match_pick (FI_EPP_LIB=fusioninfer_b200/lib/libfi_epp_timing.so FI_EPP_VERBOSE=1)
TIMING_LIB := fusioninfer_b200/lib/libfi_epp_timing.so
timing: $(TIMING_LIB)
$(TIMING_LIB): $(CU_SRCS) $(HDRS) $(OBJDIR)/epp_config.o
	@mkdir -p $(OBJDIR)/timing
	for f in $(CU_SRCS); do $(NVCC) $(ARCH) -O3 -std=c++17 -lineinfo -DFI_MATCH_TIMING -Xcompiler -fPIC -c $$f -o $(OBJDIR)/timing/$$(basename $$f .cu).o || exit 1; done
	$(NVCC) $(ARCH) -shared -o $@ $(OBJDIR)/timing/*.o $(OBJDIR)/epp_config.o -ldl
.PHONY: timing

# A/B builds of the library with extra defines:  make variant NAME=b16 DEFS=-DFI_MATCH_BATCH=16
# -> fusioninfer_b200/lib/libfi_epp_$(NAME).so (select it with FI_EPP_LIB=<path>)
variant: $(CU_SRCS) $(HDRS) $(OBJDIR)/epp_config.o
	@mkdir -p $(OBJDIR)/$(NAME)
	for f in $(CU_SRCS); do $(NVCC) $(ARCH) -O3 -std=c++17 -lineinfo $(DEFS) -Xcompiler -fPIC -c $$f -o $(OBJDIR)/$(NAME)/$$(basename $$f .cu).o || exit 1; done
	$(NVCC) $(ARCH) -shared -o fusioninfer_b200/lib/libfi_epp_$(NAME).so $(OBJDIR)/$(NAME)/*.o $(OBJDIR)/epp_config.o -ldl
.PHONY: variant
