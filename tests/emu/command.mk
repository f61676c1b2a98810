# CPU block emulator of the orientation and command kernels (TEST INFRASTRUCTURE; see cuda_emu.h).  g++ only; no contraction into FMA,
# as the library compiles a1mpc_command.cu (--fmad=false).
#   make -f command.mk        (tests/emu/emu_command_py.py runs it)
CXX ?= g++
CSRC := ../../a1-qp-mpc-controller_b200/csrc
liba1mpc_emu_command.so: emu_command.cpp cuda_emu.cpp cuda_emu.h $(CSRC)/a1mpc_command.cuh $(CSRC)/a1mpc_filter.cuh $(CSRC)/a1mpc_device.cuh ../../include/a1mpc.h
	$(CXX) -std=c++17 -O1 -mfma -march=x86-64-v3 -ffp-contract=off -fPIC -shared -Wno-unknown-pragmas -Wno-attributes -o $@ emu_command.cpp cuda_emu.cpp -lpthread -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_emu_command.so
