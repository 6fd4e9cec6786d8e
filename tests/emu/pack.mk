# TEST INFRASTRUCTURE. The CPU oracle with the frame packer's host build (kernels/pack.cuh) and the planner's write plan
# (host/planner.cc plan_write): every output layout of a frame computed on the CPU, for tests/test_write_layouts.py:
# make -f pack.mk.
CXX ?= g++
CUDA_INC ?= /usr/local/cuda/include
CXXFLAGS ?= -std=c++17 -O2 -fPIC -Wall -Wno-unused-function -Wno-unused-variable -Wno-unknown-pragmas -ffp-contract=off -fno-fast-math -pthread
CSRC := ../../jxl_oxide_b200/csrc
HOST := $(CSRC)/host
KERN := $(CSRC)/kernels
ORA := ../../oracle
SRCS := pack_capi.cc $(ORA)/oracle_modular.cc $(ORA)/oracle_vardct.cc $(ORA)/oracle_render.cc \
        $(HOST)/entropy.cc $(HOST)/headers.cc $(HOST)/modular_syntax.cc $(HOST)/frame_syntax.cc $(HOST)/planner.cc $(HOST)/icc.cc
OUT := _build/libjxlpack.so

$(OUT): $(SRCS) cuda_shim.h $(KERN)/pack.cuh $(KERN)/pixel_math.cuh $(KERN)/kernels.h $(wildcard $(ORA)/*.h) $(wildcard $(HOST)/*.h) $(wildcard $(HOST)/*.inc)
	@mkdir -p _build
	$(CXX) $(CXXFLAGS) -I$(CUDA_INC) -shared -o $@ $(SRCS)

clean:
	rm -f $(OUT)
