# CPU block emulator of the warm-started scheduled kernels (TEST INFRASTRUCTURE; see cuda_emu.h).  g++ only.
#   make -f ext_warm.mk        (tests/emu/emu_ext_warm_py.py runs it)
CXX ?= g++
CSRC := ../../a1-qp-mpc-controller_b200/csrc
liba1mpc_emu_ext_warm.so: emu_ext_warm.cpp cuda_emu.cpp cuda_emu.h $(CSRC)/a1mpc_device.cuh $(CSRC)/a1mpc_solve_body.inc $(CSRC)/a1mpc_sched.cuh $(CSRC)/a1mpc_sched_body.inc $(CSRC)/a1mpc_misc.cuh ../../include/a1mpc.h
	$(CXX) -std=c++17 -O1 -mfma -march=x86-64-v3 -fPIC -shared -Wno-unknown-pragmas -Wno-attributes -o $@ emu_ext_warm.cpp cuda_emu.cpp -lpthread -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_emu_ext_warm.so
