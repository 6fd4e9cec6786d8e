# TEST INFRASTRUCTURE. The oracle library rebuilt around EmuBackend (emu_backend.cc) like Makefile, with the SIMT model of
# every number of HF streams per warp (lanes_k_emu.cc): make -f lanes_k.mk.
CXX ?= g++
CUDA_INC ?= /usr/local/cuda/include
CXXFLAGS ?= -std=c++17 -O2 -ftree-vectorize -fvect-cost-model=dynamic -fPIC -Wall -Wno-unused-function -Wno-unused-variable -Wno-unknown-pragmas -ffp-contract=off -fno-fast-math -pthread
CSRC := ../../jxl_oxide_b200/csrc
HOST := $(CSRC)/host
KERN := $(CSRC)/kernels
ORA := ../../oracle
SRCS := lanes_k_emu.cc launch_tables_host.cc $(ORA)/oracle_capi.cc $(ORA)/oracle_modular.cc $(ORA)/oracle_vardct.cc $(ORA)/oracle_render.cc \
        $(HOST)/entropy.cc $(HOST)/headers.cc $(HOST)/modular_syntax.cc $(HOST)/frame_syntax.cc $(HOST)/planner.cc $(HOST)/icc.cc
OUT := _build/libjxlemu_lanes_k.so

$(OUT): $(SRCS) emu_backend.cc cuda_shim.h host_sink.h $(CSRC)/launch_tables.h $(CSRC)/launch_tables.cc $(wildcard $(KERN)/*.cuh) $(KERN)/kernels.h $(wildcard $(ORA)/*.h) $(wildcard $(HOST)/*.h) $(wildcard $(HOST)/*.inc)
	@mkdir -p _build
	$(CXX) $(CXXFLAGS) -I$(CUDA_INC) -DJXLO_BACKEND_FACTORY=make_lanes_k_backend -shared -Wl,-Bsymbolic -o $@ $(SRCS)

clean:
	rm -f $(OUT)
