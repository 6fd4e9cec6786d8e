# TEST INFRASTRUCTURE. The JPEG-reconstruction oracle rebuilt with the host emulation of the device scan encoder
# (jpeg_emu.cc: the per-block code of kernels/jpeg_blocks.cuh run in launch order): make -f jpeg.mk.
CXX ?= g++
CXXFLAGS ?= -std=c++17 -O2 -ftree-vectorize -fvect-cost-model=dynamic -fPIC -Wall -Wno-unused-function -ffp-contract=off -fno-fast-math -pthread
CSRC := ../../jxl_oxide_b200/csrc
HOST := $(CSRC)/host
ORA := ../../oracle
SRCS := jpeg_emu.cc $(ORA)/oracle_jbr.cc $(ORA)/oracle_modular.cc $(ORA)/oracle_vardct.cc $(ORA)/oracle_render.cc \
        $(HOST)/entropy.cc $(HOST)/headers.cc $(HOST)/modular_syntax.cc $(HOST)/frame_syntax.cc $(HOST)/planner.cc $(HOST)/icc.cc \
        $(HOST)/jbrd.cc
OUT := _build/libjxlejpeg.so

$(OUT): $(SRCS) $(CSRC)/kernels/jpeg_blocks.cuh $(wildcard $(ORA)/*.h) $(wildcard $(HOST)/*.h) $(wildcard $(HOST)/*.inc)
	@mkdir -p _build
	$(CXX) $(CXXFLAGS) -shared -Wl,--no-undefined -o $@ $(SRCS) -ldl

clean:
	rm -f $(OUT)
