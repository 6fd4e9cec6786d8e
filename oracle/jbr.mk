# TEST INFRASTRUCTURE. Builds the JPEG-reconstruction oracle (oracle_jbr.cc: the scalar sequential scan encoder over the
# oracle's own decode) as a shared library for ctypes: make -f jbr.mk. Same flags as the oracle's Makefile.
CXX ?= g++
CXXFLAGS ?= -std=c++17 -O2 -ftree-vectorize -fvect-cost-model=dynamic -fPIC -Wall -ffp-contract=off -fno-fast-math -pthread
HOST := ../jxl_oxide_b200/csrc/host
SRCS := oracle_jbr.cc oracle_modular.cc oracle_vardct.cc oracle_render.cc \
        $(HOST)/entropy.cc $(HOST)/headers.cc $(HOST)/modular_syntax.cc $(HOST)/frame_syntax.cc $(HOST)/planner.cc $(HOST)/icc.cc \
        $(HOST)/jbrd.cc
OUT := _build/libjxlojbr.so

$(OUT): $(SRCS) oracle_backend.h oracle_tables.h oracle_jbr.h $(wildcard $(HOST)/*.h) $(wildcard $(HOST)/*.inc) \
        ../jxl_oxide_b200/csrc/kernels/jpeg_blocks.cuh
	@mkdir -p _build
	$(CXX) $(CXXFLAGS) -shared -Wl,--no-undefined -o $@ $(SRCS) -ldl

clean:
	rm -f $(OUT)
