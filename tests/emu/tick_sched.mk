# CPU block emulator of the scheduled tick's front kernel (TEST INFRASTRUCTURE; see cuda_emu.h): tick_front_sched next to the kinematics,
# update_plan and swing kernels it fuses, with the flags of tick.mk's liba1mpc_emu_tick_b.so.  A library of its own, because every header
# defines its kernels for exactly one translation unit.
#   make -f tick_sched.mk        (tests/emu/emu_tick_sched_py.py runs it)
CXX ?= g++
CSRC := ../../a1-qp-mpc-controller_b200/csrc
FLAGS := -std=c++17 -O1 -mfma -march=x86-64-v3 -fPIC -shared -Wno-unknown-pragmas -Wno-attributes
all: liba1mpc_emu_tick_sched.so
liba1mpc_emu_tick_sched.so: emu_tick_sched.cpp cuda_emu.cpp cuda_emu.h $(CSRC)/a1mpc_tick.cuh $(CSRC)/a1mpc_estim.cuh $(CSRC)/a1mpc_misc.cuh $(CSRC)/a1mpc_swing.cuh $(CSRC)/a1mpc_filter.cuh $(CSRC)/a1mpc_device.cuh ../../include/a1mpc.h
	$(CXX) $(FLAGS) -o $@ emu_tick_sched.cpp cuda_emu.cpp -lpthread -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_emu_tick_sched.so
.PHONY: all clean
