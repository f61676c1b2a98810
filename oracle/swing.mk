# Test infrastructure of the swing-leg / terrain-pitch stage, next to the main oracle Makefile:
#   all: liba1mpc_swing_oracle.so, the oracle's restatement (swing_oracle.cpp)
#   ref: where /root/reference is mounted, _ref/libref_swing.so -- the REFERENCE'S OWN sources compiled unmodified from where they lie
#        against the header stand-ins in ref_shim/, with the multi-tick driver ref_swing_wrap.cpp (outputs under _ref/ only, git-ignored)
#   make -C oracle -f swing.mk all ref        (the top-level Makefile runs it)
CXX ?= g++
CXXFLAGS ?= -O3 -march=x86-64-v3 -std=c++17 -fPIC -Wall -Wextra -Wno-unused-parameter
all: liba1mpc_swing_oracle.so
liba1mpc_swing_oracle.so: swing_oracle.cpp
	$(CXX) $(CXXFLAGS) -shared -o $@ swing_oracle.cpp -l:libstdc++.so.6 -lm
REF ?= /root/reference/src/a1_cpp/src
REFINC := -I ref_shim -I ref_shim/eigen3 -I $(REF)
REFFLAGS := -O2 -std=c++17 -fPIC -w $(REFINC)
REFSRC := $(REF)/ConvexMpc.cpp $(REF)/A1RobotControl.cpp $(REF)/A1BasicEKF.cpp $(REF)/utils/Utils.cpp $(REF)/legKinematics/A1Kinematics.cpp
SHIM := $(shell find ref_shim -type f)
ref:
	@if [ -f $(REF)/A1RobotControl.cpp ]; then $(MAKE) -s -f swing.mk _ref/libref_swing.so; \
	else echo "oracle/_ref/libref_swing.so: reference sources not present, skipped"; fi
_ref/libref_swing.so: ref_swing_wrap.cpp $(SHIM)
	@mkdir -p _ref
	$(CXX) $(REFFLAGS) -shared -o $@ ref_swing_wrap.cpp $(REFSRC) -l:libstdc++.so.6 -lm
clean:
	rm -f liba1mpc_swing_oracle.so _ref/libref_swing.so
.PHONY: all ref clean
