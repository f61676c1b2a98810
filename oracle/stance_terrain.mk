# Test infrastructure of the stance QP on terrain normals, next to the main oracle Makefile:
#   all: liba1mpc_stance_terrain_oracle.so, the 12-force QP of oracle_grf_qp_single in per-foot terrain frames (stance_terrain_oracle.cpp)
#   make -C oracle -f stance_terrain.mk all        (the top-level Makefile runs it, after the main oracle)
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -Wall -Wextra -Wno-unused-parameter
all: liba1mpc_stance_terrain_oracle.so
liba1mpc_stance_terrain_oracle.so: stance_terrain_oracle.cpp liba1mpc_oracle.so ../include/a1mpc.h
	$(CXX) $(CXXFLAGS) -shared -o $@ stance_terrain_oracle.cpp -L. -la1mpc_oracle -Wl,-rpath,'$$ORIGIN' -lpthread -l:libstdc++.so.6 -lm
liba1mpc_oracle.so:
	$(MAKE) -s liba1mpc_oracle.so
clean:
	rm -f liba1mpc_stance_terrain_oracle.so
.PHONY: all clean
