# Builds coslam_b200/libcoslam_b200.so (hand-written CUDA for sm_90a behind the C-ABI) and the
# CPU oracle.  `make` here is what __graft_entry__.build() runs.
NVCC ?= /usr/local/cuda/bin/nvcc
HOSTCXX := /usr/bin/g++
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := $(ARCH) -O3 -lineinfo -std=c++17 -ccbin $(HOSTCXX) -Xcompiler -fPIC,-Wall,-Wno-unknown-pragmas \
           -Xptxas -v --expt-relaxed-constexpr
CSRC := coslam_b200/csrc
OBJS := $(CSRC)/common.o $(CSRC)/klt.o $(CSRC)/pose.o $(CSRC)/ba.o $(CSRC)/posegraph.o
LIB := coslam_b200/libcoslam_b200.so

all: $(LIB) oracle

$(CSRC)/pose.o: NVFLAGS += -fmad=false
# LK solve is tolerance-parity: approximate sqrt/div there; bit-exact kernels use explicit _rn intrinsics
$(CSRC)/klt.o: NVFLAGS += -prec-sqrt=false -prec-div=false

$(CSRC)/%.o: $(CSRC)/%.cu $(wildcard $(CSRC)/*.cuh) include/coslam_b200.h
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> $(@:.o=.ptxas.log) || (cat $(@:.o=.ptxas.log); exit 1)

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -ldl

oracle:
	$(MAKE) -s -C oracle
	$(MAKE) -s -C oracle -f Makefile.pg_general

clean:
	rm -f $(CSRC)/*.o $(CSRC)/*.ptxas.log $(LIB)
	$(MAKE) -C oracle clean
	$(MAKE) -C oracle -f Makefile.pg_general clean

.PHONY: all oracle clean
