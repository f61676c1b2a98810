# CPU block emulator of the swing-leg and terrain-pitch kernels (TEST INFRASTRUCTURE; see cuda_emu.h).  g++ only.
#   make -f swing.mk        (tests/emu/emu_swing_py.py runs it)
CXX ?= g++
CSRC := ../../a1-qp-mpc-controller_b200/csrc
liba1mpc_emu_swing.so: emu_swing.cpp cuda_emu.cpp cuda_emu.h $(CSRC)/a1mpc_swing.cuh $(CSRC)/a1mpc_device.cuh ../../include/a1mpc.h
	$(CXX) -std=c++17 -O1 -mfma -march=x86-64-v3 -fPIC -shared -Wno-unknown-pragmas -Wno-attributes -o $@ emu_swing.cpp cuda_emu.cpp -lpthread -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_emu_swing.so
