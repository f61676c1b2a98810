# CPU block emulator of the a1mpc_solve_dense_batch and a1mpc_grf_qp_batch kernels (TEST INFRASTRUCTURE; see cuda_emu.h).  g++ only.
#   make -f dense.mk        (tests/emu/emu_dense_py.py runs it)
CXX ?= g++
CSRC := ../../a1-qp-mpc-controller_b200/csrc
liba1mpc_emu_dense.so: emu_dense.cpp cuda_emu.cpp cuda_emu.h $(CSRC)/a1mpc_dense.cu $(CSRC)/a1mpc_device.cuh ../../include/a1mpc.h
	$(CXX) -std=c++17 -O1 -mfma -march=x86-64-v3 -fPIC -shared -Wno-unknown-pragmas -Wno-attributes -o $@ emu_dense.cpp cuda_emu.cpp -lpthread -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_emu_dense.so
