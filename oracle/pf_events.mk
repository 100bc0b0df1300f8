# TEST INFRASTRUCTURE ONLY — the checkers of the resident set's odometry-noise redraw, expansion noise and IMU gravity
# update, beside Makefile's (same compiler, flags and reference location, taken from it):
#   make -f pf_events.mk                  -> libmcl3dl_pf_events_oracle.so  (port; always buildable)
#   make -f pf_events.mk pf-events-ref    -> _ref/libmcl3dl_pf_events_ref.so (the reference's own filter, State6DOF and
#                                            ImuMeasurementModelGravity, header-only)
#   make -f pf_events.mk pf-events-parity -> _ref/pf_events_parity_test (resident cycles with IMU updates between clouds,
#                                            the redraw and expansion resetting through the C++ adapter vs the reference
#                                            filter fed the same draws; an H100 runs it, tests/test_gpu_pf_events.py)
include Makefile
.DEFAULT_GOAL := pf-events-port

PFE_CXXFLAGS = $(CXXFLAGS) -Wno-subobject-linkage
REF_SOURCES = $(REFERENCE)/src/lidar_measurement_model_likelihood.cpp $(REFERENCE)/src/lidar_measurement_model_beam.cpp

pf-events-port: libmcl3dl_pf_events_oracle.so

libmcl3dl_pf_events_oracle.so: pf_events_oracle.cpp pf_events_api.h ../include/mcl3dl_b200.h
	$(CXX) $(PFE_CXXFLAGS) -shared -o $@ pf_events_oracle.cpp

pf-events-ref: _ref/libmcl3dl_pf_events_ref.so

_ref/libmcl3dl_pf_events_ref.so: pf_events_ref_driver.cpp pf_events_api.h ../include/mcl3dl_b200.h $(wildcard shim/*/*.h shim/*/*/*.h shim/Eigen/Core)
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(PFE_CXXFLAGS) -Ishim -I$(REFERENCE)/include -shared -o $@ pf_events_ref_driver.cpp

pf-events-parity: _ref/pf_events_parity_test

_ref/pf_events_parity_test: pf_events_parity_test.cpp ../mcl_3dl_b200/host/lidar_measurement_model_b200.h ../include/mcl3dl_b200.h ../mcl_3dl_b200/libmcl3dl_b200.so
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -fPIE -DPCL_NO_PRECOMPILE -Ishim -I$(REFERENCE)/include -I../include -o $@ pf_events_parity_test.cpp \
	    $(REF_SOURCES) -L../mcl_3dl_b200 -lmcl3dl_b200 -Wl,-rpath,'$$ORIGIN/../../mcl_3dl_b200'

.PHONY: pf-events-port pf-events-ref pf-events-parity
