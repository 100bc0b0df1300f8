# TEST INFRASTRUCTURE ONLY — the checkers of the resident set's landmark update, odometry-error reset and published
# poses, beside Makefile's (same compiler, flags and reference location, taken from it):
#   make -f pf_landmark.mk                    -> libmcl3dl_pf_landmark_oracle.so  (port; always buildable)
#   make -f pf_landmark.mk pf-landmark-ref    -> _ref/libmcl3dl_pf_landmark_ref.so (the reference's own filter, State6DOF
#                                               and Quat, header-only)
#   make -f pf_landmark.mk landmark-parity    -> _ref/landmark_parity_test (a resident cycle, cbLandmark, a pose-jump
#                                               reset and the published poses through the C++ adapter vs the reference
#                                               filter; an H100 runs it, tests/test_gpu_pf_landmark.py).  Compiled against
#                                               shim_nd/ first: the reference's NormalLikelihoodNd needs a 6x6 matrix.
include Makefile
.DEFAULT_GOAL := pf-landmark-port

PFL_CXXFLAGS = $(CXXFLAGS) -Wno-subobject-linkage
REF_SOURCES = $(REFERENCE)/src/lidar_measurement_model_likelihood.cpp $(REFERENCE)/src/lidar_measurement_model_beam.cpp

pf-landmark-port: libmcl3dl_pf_landmark_oracle.so

libmcl3dl_pf_landmark_oracle.so: pf_landmark_oracle.cpp pf_landmark_api.h ../include/mcl3dl_b200.h
	$(CXX) $(PFL_CXXFLAGS) -shared -o $@ pf_landmark_oracle.cpp

pf-landmark-ref: _ref/libmcl3dl_pf_landmark_ref.so

_ref/libmcl3dl_pf_landmark_ref.so: pf_landmark_ref_driver.cpp pf_landmark_api.h ../include/mcl3dl_b200.h $(wildcard shim/*/*.h shim/*/*/*.h shim/Eigen/Core)
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(PFL_CXXFLAGS) -Ishim -I$(REFERENCE)/include -shared -o $@ pf_landmark_ref_driver.cpp

landmark-parity: _ref/landmark_parity_test

_ref/landmark_parity_test: landmark_parity_test.cpp ../mcl_3dl_b200/host/lidar_measurement_model_b200.h ../include/mcl3dl_b200.h ../mcl_3dl_b200/libmcl3dl_b200.so shim_nd/Eigen/Core shim_nd/Eigen/LU
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -fPIE -DPCL_NO_PRECOMPILE -Ishim_nd -Ishim -I$(REFERENCE)/include -I../include -o $@ landmark_parity_test.cpp \
	    $(REF_SOURCES) -L../mcl_3dl_b200 -lmcl3dl_b200 -Wl,-rpath,'$$ORIGIN/../../mcl_3dl_b200'

.PHONY: pf-landmark-port pf-landmark-ref landmark-parity
