# CPU block emulator of the terrain stage with normals (TEST INFRASTRUCTURE; see cuda_emu.h): terrain_normals_kernel of a1mpc_swing.cuh
# next to terrain_pitch_kernel, whose stage it repeats, and the kernels that fill the swing state.  The flags of swing.mk.
#   make -f terrain_normals.mk        (tests/emu/emu_terrain_normals_py.py runs it)
CXX ?= g++
CSRC := ../../a1-qp-mpc-controller_b200/csrc
FLAGS := -std=c++17 -O1 -mfma -march=x86-64-v3 -fPIC -shared -Wno-unknown-pragmas -Wno-attributes
all: liba1mpc_emu_terrain_normals.so
liba1mpc_emu_terrain_normals.so: emu_terrain_normals.cpp cuda_emu.cpp cuda_emu.h $(CSRC)/a1mpc_swing.cuh $(CSRC)/a1mpc_filter.cuh $(CSRC)/a1mpc_device.cuh ../../include/a1mpc.h
	$(CXX) $(FLAGS) -o $@ emu_terrain_normals.cpp cuda_emu.cpp -lpthread -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_emu_terrain_normals.so
.PHONY: all clean
