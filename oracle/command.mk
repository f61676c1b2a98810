# Test infrastructure of the orientation / command stages, next to the main oracle Makefile:
#   all: liba1mpc_command_oracle.so, the oracle's restatement (command_oracle.cpp)
#   ref: where /root/reference is mounted, _ref/libref_command.so -- the REFERENCE'S OWN utils/Utils.cpp compiled unmodified from where
#        it lies against the header stand-ins in ref_shim/, with ref_command_wrap.cpp (its MovingWindowFilter is header-only)
#   make -C oracle -f command.mk all ref        (the top-level Makefile runs it)
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -ffp-contract=off -std=c++17 -fPIC -Wall -Wextra -Wno-unused-parameter
all: liba1mpc_command_oracle.so
liba1mpc_command_oracle.so: command_oracle.cpp
	$(CXX) $(CXXFLAGS) -shared -o $@ command_oracle.cpp -l:libstdc++.so.6 -lm
REF ?= /root/reference/src/a1_cpp/src
REFINC := -I ref_shim -I ref_shim/eigen3 -I $(REF)
REFFLAGS := -O2 -std=c++17 -fPIC -w $(REFINC)
SHIM := $(shell find ref_shim -type f)
ref:
	@if [ -f $(REF)/utils/Utils.cpp ]; then $(MAKE) -s -f command.mk _ref/libref_command.so; \
	else echo "oracle/_ref/libref_command.so: reference sources not present, skipped"; fi
_ref/libref_command.so: ref_command_wrap.cpp $(SHIM)
	@mkdir -p _ref
	$(CXX) $(REFFLAGS) -shared -o $@ ref_command_wrap.cpp $(REF)/utils/Utils.cpp -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_command_oracle.so _ref/libref_command.so
.PHONY: all ref clean
