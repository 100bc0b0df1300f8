# TEST INFRASTRUCTURE ONLY — the adapter parity program of the map intake (mcl3dl_map_load / mcl3dl_map_update_*),
# beside Makefile's (same compiler, flags and reference location, taken from it):
#   make -f map_intake.mk map-intake-parity -> _ref/map_intake_parity_test (the node's map callbacks on its restated host
#                                    path and through the C++ adapter's loadMapMessage / loadMapCloud / setMapUpdate /
#                                    commitMapUpdate / clearMapUpdate / mapCloud, with the reference's own models; an H100
#                                    runs it, tests/test_gpu_map_intake.py)
include Makefile
.DEFAULT_GOAL := map-intake-parity

REF_SOURCES = $(REFERENCE)/src/lidar_measurement_model_likelihood.cpp $(REFERENCE)/src/lidar_measurement_model_beam.cpp

map-intake-parity: _ref/map_intake_parity_test

_ref/map_intake_parity_test: map_intake_parity_test.cpp ../mcl_3dl_b200/host/lidar_measurement_model_b200.h ../include/mcl3dl_b200.h ../mcl_3dl_b200/libmcl3dl_b200.so shim/sensor_msgs/PointCloud2.h ../tests/hostsim/scan_hostsim.cpp ../mcl_3dl_b200/csrc/scan_funcs.cuh
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -fPIE -DPCL_NO_PRECOMPILE -Ishim -I$(REFERENCE)/include -I../include -o $@ map_intake_parity_test.cpp \
	    $(REF_SOURCES) -L../mcl_3dl_b200 -lmcl3dl_b200 -Wl,-rpath,'$$ORIGIN/../../mcl_3dl_b200'

.PHONY: map-intake-parity
