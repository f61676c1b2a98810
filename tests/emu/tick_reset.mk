# CPU block emulator of the tick's masked reset kernels (TEST INFRASTRUCTURE; see cuda_emu.h): tick_reset_robots_kernel and ekf_init_pending
# of a1mpc_tick.cuh next to the init kernels whose per-robot bodies they share (imu_init_kernel and command_init_kernel of a1mpc_command.cuh,
# swing_init_kernel, ekf_init_kernel).  Those kernels only store values, so one library with the flags of tick.mk's liba1mpc_emu_tick_b.so
# holds both headers.
#   make -f tick_reset.mk        (tests/emu/emu_tick_reset_py.py runs it)
CXX ?= g++
CSRC := ../../a1-qp-mpc-controller_b200/csrc
FLAGS := -std=c++17 -O1 -mfma -march=x86-64-v3 -fPIC -shared -Wno-unknown-pragmas -Wno-attributes
all: liba1mpc_emu_tick_reset.so
liba1mpc_emu_tick_reset.so: emu_tick_reset.cpp cuda_emu.cpp cuda_emu.h $(CSRC)/a1mpc_tick.cuh $(CSRC)/a1mpc_command.cuh $(CSRC)/a1mpc_command_state.cuh $(CSRC)/a1mpc_estim.cuh $(CSRC)/a1mpc_misc.cuh $(CSRC)/a1mpc_swing.cuh $(CSRC)/a1mpc_filter.cuh $(CSRC)/a1mpc_device.cuh ../../include/a1mpc.h
	$(CXX) $(FLAGS) -o $@ emu_tick_reset.cpp cuda_emu.cpp -lpthread -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_emu_tick_reset.so
.PHONY: all clean
