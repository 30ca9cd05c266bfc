# Builds the C-ABI shared library for sm_90a (H100).  `make` == what __graft_entry__.build() runs.
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -Wall -Xcompiler -Wno-unused-function
SRC := cvxopt_b200/csrc
OBJ := $(SRC)/gemm_dmma.o $(SRC)/chol.o $(SRC)/cone.o $(SRC)/kkt_api.o $(SRC)/blocks_api.o $(SRC)/batch_ipm.o $(SRC)/cone_vec.o $(SRC)/ozaki_syrk.o $(SRC)/nt_scaling.o $(SRC)/kkt_qr.o $(SRC)/kkt_ldl.o $(SRC)/kkt_sparse.o
LIB := cvxopt_b200/libcvxopt_b200.so
# CPython extension mirroring cvxopt.misc_solvers over the C ABI (host side of the drop-in boundary)
PYTHON ?= python
PYINC := $(shell $(PYTHON) -c "import sysconfig; print(sysconfig.get_paths()['include'])")
PYEXT := $(shell $(PYTHON) -c "import sysconfig; print(sysconfig.get_config_var('EXT_SUFFIX'))")
EXT := cvxopt_b200/_misc_solvers$(PYEXT)

all: $(LIB) $(EXT) tools/dmma_rate tools/syrk_feed

$(EXT): $(SRC)/_misc_solvers.c include/cvxopt_b200.h $(LIB)
	gcc -O2 -fPIC -shared -Wall -I$(PYINC) $< -o $@ -Lcvxopt_b200 -lcvxopt_b200 -Wl,-rpath,'$$ORIGIN'

$(SRC)/%.o: $(SRC)/%.cu $(SRC)/common.cuh $(SRC)/cone.cuh $(SRC)/kkt_internal.cuh include/cvxopt_b200.h
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(LIB): $(OBJ)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJ) -lcudart

# standalone probe of the fp64 mma.sync shapes (fragment layouts, issue rate); see tools/README.md
tools/dmma_rate: tools/dmma_rate.cu
	$(NVCC) $(ARCH) -O3 -std=c++17 -o $@ $<

# standalone probe of the SYRK's L2 -> shared-memory operand feed (no DMMAs); see tools/README.md
tools/syrk_feed: tools/syrk_feed.cu
	$(NVCC) $(ARCH) -O3 -std=c++17 -o $@ $<

clean:
	rm -f $(OBJ) $(LIB) $(EXT) tools/dmma_rate tools/syrk_feed
.PHONY: all clean
