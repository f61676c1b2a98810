# CPU block emulator of the two fused kernels of a control tick (TEST INFRASTRUCTURE; see cuda_emu.h), each next to the staged kernels it
# fuses and with their flags: tick_front_a with the orientation and command kernels, no contraction into FMA (command.mk; the library
# compiles a1mpc_command.cu with --fmad=false); tick_front_b with the kinematics, update_plan and swing kernels, the flags of swing.mk.
# Two libraries, because every header defines its kernels for exactly one translation unit.
#   make -f tick.mk        (tests/emu/emu_tick_py.py runs it)
CXX ?= g++
CSRC := ../../a1-qp-mpc-controller_b200/csrc
FLAGS := -std=c++17 -O1 -mfma -march=x86-64-v3 -fPIC -shared -Wno-unknown-pragmas -Wno-attributes
all: liba1mpc_emu_tick_a.so liba1mpc_emu_tick_b.so
liba1mpc_emu_tick_a.so: emu_tick.cpp cuda_emu.cpp cuda_emu.h $(CSRC)/a1mpc_command.cuh $(CSRC)/a1mpc_filter.cuh $(CSRC)/a1mpc_device.cuh ../../include/a1mpc.h
	$(CXX) $(FLAGS) -ffp-contract=off -DEMU_TICK_PART=1 -o $@ emu_tick.cpp cuda_emu.cpp -lpthread -l:libstdc++.so.6 -lm
liba1mpc_emu_tick_b.so: emu_tick.cpp cuda_emu.cpp cuda_emu.h $(CSRC)/a1mpc_tick.cuh $(CSRC)/a1mpc_estim.cuh $(CSRC)/a1mpc_misc.cuh $(CSRC)/a1mpc_swing.cuh $(CSRC)/a1mpc_filter.cuh $(CSRC)/a1mpc_device.cuh ../../include/a1mpc.h
	$(CXX) $(FLAGS) -DEMU_TICK_PART=2 -o $@ emu_tick.cpp cuda_emu.cpp -lpthread -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_emu_tick_a.so liba1mpc_emu_tick_b.so
.PHONY: all clean
