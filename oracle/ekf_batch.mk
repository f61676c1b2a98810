# Test infrastructure of the batched Kalman filter, next to the main oracle Makefile:
#   all: liba1mpc_ekf_batch_oracle.so, oracle_ekf_update of liba1mpc_oracle.so over a batch on host threads (ekf_batch_oracle.cpp)
#   make -C oracle -f ekf_batch.mk all        (the top-level Makefile runs it, after the main oracle)
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -Wall -Wextra -Wno-unused-parameter
all: liba1mpc_ekf_batch_oracle.so
liba1mpc_ekf_batch_oracle.so: ekf_batch_oracle.cpp liba1mpc_oracle.so
	$(CXX) $(CXXFLAGS) -shared -o $@ ekf_batch_oracle.cpp -L. -la1mpc_oracle -Wl,-rpath,'$$ORIGIN' -lpthread -l:libstdc++.so.6 -lm
liba1mpc_oracle.so:
	$(MAKE) -s liba1mpc_oracle.so
clean:
	rm -f liba1mpc_ekf_batch_oracle.so
.PHONY: all clean
