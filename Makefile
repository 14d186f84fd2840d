# vartrix_b200 -- build the sm_90a (H100) engine library (and the oracle used by the tests).
NVCC      ?= /usr/local/cuda/bin/nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
EXTRA     ?=
NVCCFLAGS := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall,-Wextra -Xptxas -v $(EXTRA)
CSRC      := vartrix_b200/csrc
LIBDIR    := vartrix_b200/lib
LIB       := $(LIBDIR)/libvartrix_b200.so

CLI       := vartrix_b200/bin/vartrix_b200
HOSTSRC   := $(CSRC)/host

all: $(LIB) $(CLI) oracle

$(LIB): $(CSRC)/vtx_api.cu $(wildcard $(CSRC)/*.cuh) include/vartrix_b200.h
	@mkdir -p $(LIBDIR)
	$(NVCC) $(NVCCFLAGS) -shared -o $@.tmp $(CSRC)/vtx_api.cu -ldl 2> $(LIBDIR)/ptxas.log || (cat $(LIBDIR)/ptxas.log; exit 1)
	@mv -f $@.tmp $@          # a tree snapshot never sees a half-written library
	@grep -E "error|warning" $(LIBDIR)/ptxas.log | grep -v "ptxas info" || true

# C++ host: BAM/VCF/FASTA decode + staging + CLI with the vartrix flag surface, on top of the C ABI
$(CLI): $(HOSTSRC)/main.cpp $(HOSTSRC)/stager.hpp $(HOSTSRC)/inputs.hpp $(HOSTSRC)/bam_reader.hpp $(HOSTSRC)/inflate_fast.hpp $(HOSTSRC)/crc32_fast.hpp $(CSRC)/vtx_record.cuh $(CSRC)/vtx_donors.cuh $(CSRC)/vtx_clusters.cuh $(CSRC)/vtx_ambient.cuh $(CSRC)/vtx_cluster_gt.cuh $(CSRC)/vtx_cluster_refine.cuh include/vartrix_b200.h $(LIB)
	@mkdir -p vartrix_b200/bin
	g++ -O2 -std=c++17 -Wall -Wextra -o $@.tmp $(HOSTSRC)/main.cpp -L$(LIBDIR) -lvartrix_b200 -lz -lpthread -Wl,-rpath,'$$ORIGIN/../lib'
	@mv -f $@.tmp $@

oracle:
	$(MAKE) -s -C oracle

clean:
	rm -f $(LIB) $(LIBDIR)/ptxas.log $(CLI)
	$(MAKE) -s -C oracle clean

.PHONY: all oracle clean
