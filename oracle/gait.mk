# Test infrastructure of the per-robot gaits, next to the main oracle Makefile:
#   ref: where /root/reference is mounted, _ref/libref_gait.so -- the REFERENCE'S OWN sources compiled unmodified from where they lie
#        against the header stand-ins in ref_shim/, with the per-robot-gait driver ref_gait_wrap.cpp (outputs under _ref/ only, git-ignored)
#   make -C oracle -f gait.mk ref        (the top-level Makefile runs it)
CXX ?= g++
REF ?= /root/reference/src/a1_cpp/src
REFINC := -I ref_shim -I ref_shim/eigen3 -I $(REF)
REFFLAGS := -O2 -std=c++17 -fPIC -w $(REFINC)
REFSRC := $(REF)/ConvexMpc.cpp $(REF)/A1RobotControl.cpp $(REF)/A1BasicEKF.cpp $(REF)/utils/Utils.cpp $(REF)/legKinematics/A1Kinematics.cpp
SHIM := $(shell find ref_shim -type f)
all:
ref:
	@if [ -f $(REF)/A1RobotControl.cpp ]; then $(MAKE) -s -f gait.mk _ref/libref_gait.so; \
	else echo "oracle/_ref/libref_gait.so: reference sources not present, skipped"; fi
_ref/libref_gait.so: ref_gait_wrap.cpp $(SHIM)
	@mkdir -p _ref
	$(CXX) $(REFFLAGS) -shared -o $@ ref_gait_wrap.cpp $(REFSRC) -l:libstdc++.so.6 -lm
clean:
	rm -f _ref/libref_gait.so
.PHONY: all ref clean
