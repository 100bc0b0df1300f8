# TEST INFRASTRUCTURE ONLY — the adapter parity program of the cloud accumulation (mcl3dl_scan_accumulate), beside
# Makefile's (same compiler, flags and reference location, taken from it):
#   make -f accum.mk accum-parity -> _ref/accum_parity_test (the reference's own CloudAccumulationLogic driving the node's
#                                    restated host path and the C++ adapter's accumulateCloud / clearAccumulated /
#                                    prepareAccumulated; an H100 runs it, tests/test_gpu_scan_accum.py)
include Makefile
.DEFAULT_GOAL := accum-parity

REF_SOURCES = $(REFERENCE)/src/cloud_accum.cpp $(REFERENCE)/src/lidar_measurement_model_likelihood.cpp \
              $(REFERENCE)/src/lidar_measurement_model_beam.cpp

accum-parity: _ref/accum_parity_test

_ref/accum_parity_test: accum_parity_test.cpp ../mcl_3dl_b200/host/lidar_measurement_model_b200.h ../include/mcl3dl_b200.h ../mcl_3dl_b200/libmcl3dl_b200.so shim/sensor_msgs/PointCloud2.h
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -fPIE -DPCL_NO_PRECOMPILE -Ishim -I$(REFERENCE)/include -I../include -o $@ accum_parity_test.cpp \
	    $(REF_SOURCES) -L../mcl_3dl_b200 -lmcl3dl_b200 -Wl,-rpath,'$$ORIGIN/../../mcl_3dl_b200'

.PHONY: accum-parity
