# CPU block emulator of the a1mpc_stance_qp_batch_ext and a1mpc_surface_normals_batch kernels (TEST INFRASTRUCTURE; see cuda_emu.h).  g++
# only, the flags of stance.mk and terrain_normals.mk.
#   make -f stance_terrain.mk        (tests/emu/emu_stance_terrain_py.py runs it)
CXX ?= g++
CSRC := ../../a1-qp-mpc-controller_b200/csrc
liba1mpc_emu_stance_terrain.so: emu_stance_terrain.cpp cuda_emu.cpp cuda_emu.h $(CSRC)/a1mpc_dense.cu $(CSRC)/a1mpc_swing.cuh $(CSRC)/a1mpc_filter.cuh $(CSRC)/a1mpc_device.cuh ../../include/a1mpc.h
	$(CXX) -std=c++17 -O1 -mfma -march=x86-64-v3 -fPIC -shared -Wno-unknown-pragmas -Wno-attributes -o $@ emu_stance_terrain.cpp cuda_emu.cpp -lpthread -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_emu_stance_terrain.so
