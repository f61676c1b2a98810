# CPU block emulator of the multi-rate tick's kernels (TEST INFRASTRUCTURE; see cuda_emu.h): the masked pack kernels of a1mpc_misc.cuh
# (pack_due_kernel, pack_ext_due_kernel, pack_ext2_due_kernel, warm_forget_no_contact_due_kernel) next to the unmasked kernels they must
# agree with, tick_rate_kernel, tick_rate_reset_kernel and plan_forces_kernel.
#   make -f tick_rate.mk        (tests/emu/emu_tick_rate_py.py runs it)
CXX ?= g++
CSRC := ../../a1-qp-mpc-controller_b200/csrc
FLAGS := -std=c++17 -O1 -mfma -march=x86-64-v3 -fPIC -shared -Wno-unknown-pragmas -Wno-attributes
all: liba1mpc_emu_tick_rate.so
liba1mpc_emu_tick_rate.so: emu_tick_rate.cpp cuda_emu.cpp cuda_emu.h $(CSRC)/a1mpc_misc.cuh $(CSRC)/a1mpc_device.cuh ../../include/a1mpc.h
	$(CXX) $(FLAGS) -o $@ emu_tick_rate.cpp cuda_emu.cpp -lpthread -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_emu_tick_rate.so
.PHONY: all clean
