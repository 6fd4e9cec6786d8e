# TEST INFRASTRUCTURE. The CPU oracle with the keyframe index and the segment entry (host/frame_index.cc): decodes one
# keyframe from its own segment, as jxlb_decode_keyframe does, so that the segmentation is checked on the CPU:
# make -f keyframes.mk.
CXX ?= g++
CXXFLAGS ?= -std=c++17 -O2 -ftree-vectorize -fvect-cost-model=dynamic -fPIC -Wall -Wno-unused-variable -ffp-contract=off -fno-fast-math -pthread
HOST := ../../jxl_oxide_b200/csrc/host
ORA := ../../oracle
SRCS := keyframes_capi.cc $(ORA)/oracle_modular.cc $(ORA)/oracle_vardct.cc $(ORA)/oracle_render.cc \
        $(HOST)/entropy.cc $(HOST)/headers.cc $(HOST)/modular_syntax.cc $(HOST)/frame_syntax.cc $(HOST)/planner.cc $(HOST)/icc.cc \
        $(HOST)/frame_index.cc
OUT := _build/libjxlkeyframes.so

$(OUT): $(SRCS) $(wildcard $(ORA)/*.h) $(wildcard $(HOST)/*.h) $(wildcard $(HOST)/*.inc)
	@mkdir -p _build
	$(CXX) $(CXXFLAGS) -shared -o $@ $(SRCS)

clean:
	rm -f $(OUT)
