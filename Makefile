# Build libdgmesh_b200.so (hand-written sm_100a kernels behind a C-ABI) and the CPU oracle.
# `python -c "import __graft_entry__ as g; g.build()"` drives this file.
NVCC      ?= /usr/local/cuda/bin/nvcc
HOSTCC    := $(shell [ -x /usr/bin/gcc ] && echo /usr/bin/gcc || echo gcc)
OMPFLAG   := $(shell echo 'int main(){return 0;}' | $(HOSTCC) -fopenmp -x c - -o /dev/null 2>/dev/null && echo -fopenmp)
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVCCFLAGS := -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC -Xptxas -v --expt-relaxed-constexpr
CSRC      := dg-mesh_b200/csrc
LIB       := dg-mesh_b200/libdgmesh_b200.so
CU        := $(wildcard $(CSRC)/*.cu)
OBJ       := $(patsubst $(CSRC)/%.cu,build/%.o,$(CU))
HDR       := $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) include/dgmesh_b200.h

ORACLE_SRC := $(wildcard oracle/*.c)
ORACLE_LIB := oracle/liboracle.so

all: $(LIB) $(ORACLE_LIB)

build/%.o: $(CSRC)/%.cu $(HDR)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -c $< -o $@ 2> build/$*.ptxas.log || (cat build/$*.ptxas.log; exit 1)

$(LIB): $(OBJ)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJ) -lcudart -lcufft

# CPU restatement of the reference algorithm (test infrastructure only).
# -ffp-contract=off: every fused multiply-add is written explicitly (fmaf) so the
# rounding sequence is under the source's control.
$(ORACLE_LIB): $(ORACLE_SRC) $(wildcard oracle/*.h)
	$(HOSTCC) -O2 -fPIC -shared -ffp-contract=off -mfma $(OMPFLAG) -o $@ $(ORACLE_SRC) -lm

clean:
	rm -rf build $(LIB) $(ORACLE_LIB)

.PHONY: all clean
