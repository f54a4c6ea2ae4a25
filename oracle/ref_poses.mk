# ORACLE — TEST INFRASTRUCTURE ONLY.
# _ref/libvicalib_ref_poses.so: ViCalibrator::GetIntegrationPoses through the reference's own types.h and
# interpolation-buffer.h, compiled UNMODIFIED from $(REF)/include against the stand-ins in ref_shim/, as Makefile's _ref
# target builds _ref/libvicalib_ref.so (oracle/ref_poses.cc has the entry point).  Built only where the reference tree
# exists (REF=<path> overrides); elsewhere an existing build is kept as it is.  No reference source is copied.
CXX ?= g++
REF ?= /root/reference

.PHONY: all
all: $(if $(wildcard $(REF)/include/vicalib),_ref/libvicalib_ref_poses.so)
_ref/libvicalib_ref_poses.so: ref_poses.cc ref_poses.mk $(wildcard ref_shim/*/*) $(wildcard ref_shim/*/*/*)
	mkdir -p _ref
	$(CXX) -O1 -std=c++17 -fPIC -shared -I ref_shim -I $(REF)/include -I . -o $@ ref_poses.cc
