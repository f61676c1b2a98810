# CPU block emulator of the per-robot gait kernels (TEST INFRASTRUCTURE; see cuda_emu.h): a1mpc_gait.cuh's update_plan_gait_kernel,
# swing_legs_gait_kernel, tick_front_b_gait, tick_front_sched_gait and gait_check_kernel, next to the plain kernels of a1mpc_tick.cuh they
# must reproduce with trot rows, with the flags of tick.mk.
#   make -f gait.mk        (tests/emu/emu_gait_py.py runs it)
CXX ?= g++
CSRC := ../../a1-qp-mpc-controller_b200/csrc
FLAGS := -std=c++17 -O1 -mfma -march=x86-64-v3 -fPIC -shared -Wno-unknown-pragmas -Wno-attributes
all: liba1mpc_emu_gait.so
liba1mpc_emu_gait.so: emu_gait.cpp cuda_emu.cpp cuda_emu.h $(CSRC)/a1mpc_gait.cuh $(CSRC)/a1mpc_tick.cuh $(CSRC)/a1mpc_estim.cuh $(CSRC)/a1mpc_misc.cuh $(CSRC)/a1mpc_swing.cuh $(CSRC)/a1mpc_filter.cuh $(CSRC)/a1mpc_device.cuh ../../include/a1mpc.h
	$(CXX) $(FLAGS) -o $@ emu_gait.cpp cuda_emu.cpp -lpthread -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_emu_gait.so
.PHONY: all clean
