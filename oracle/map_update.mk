# TEST INFRASTRUCTURE ONLY — the node's map update against the reference models, beside Makefile's (same compiler, flags
# and reference location, taken from it):
#   make -f map_update.mk map-update-parity -> _ref/map_update_parity_test (reference models vs the C++ adapter across
#                                              cbMapUpdateTimer's appends; an H100 runs it, tests/test_gpu_map_update_parity.py)
include Makefile
.DEFAULT_GOAL := map-update-parity

map-update-parity: _ref/map_update_parity_test

_ref/map_update_parity_test: map_update_parity_test.cpp ../mcl_3dl_b200/host/lidar_measurement_model_b200.h ../include/mcl3dl_b200.h ../mcl_3dl_b200/libmcl3dl_b200.so
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -fPIE -DPCL_NO_PRECOMPILE -Ishim -I$(REFERENCE)/include -I../include -o $@ map_update_parity_test.cpp \
	    $(REFERENCE)/src/lidar_measurement_model_likelihood.cpp $(REFERENCE)/src/lidar_measurement_model_beam.cpp \
	    -L../mcl_3dl_b200 -lmcl3dl_b200 -Wl,-rpath,'$$ORIGIN/../../mcl_3dl_b200'

.PHONY: map-update-parity
