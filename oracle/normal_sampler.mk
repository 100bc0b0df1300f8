# TEST INFRASTRUCTURE ONLY — the checkers of the normal-weighted sampler (PointCloudSamplerWithNormal), beside Makefile's
# (same compiler, flags and reference location, taken from it):
#   make -f normal_sampler.mk                       -> libmcl3dl_normal_oracle.so (port; always buildable)
#   make -f normal_sampler.mk normal-ref            -> _ref/libmcl3dl_normal_ref.so (the reference's own
#                                                      PointCloudSamplerWithNormal<PointXYZIL>, header-only)
#   make -f normal_sampler.mk normal-parity         -> _ref/normal_sampler_parity_test (the adapter's
#                                                      sampleWithNormalPrepared with the reference filter's statistics vs
#                                                      the port; an H100 runs it, tests/test_gpu_normal_sampler.py)
# The reference tier and the parity program compile against shim_ns/ first (NormalEstimation, a double
# SelfAdjointEigenSolver, ros::WallTime: repo-written stand-ins over normal_eigen.h), then shim/.
include Makefile
.DEFAULT_GOAL := normal-port

REF_SOURCES = $(REFERENCE)/src/lidar_measurement_model_likelihood.cpp $(REFERENCE)/src/lidar_measurement_model_beam.cpp
SHIM_NS = shim_ns/Eigen/Core shim_ns/Eigen/Eigenvalues shim_ns/ros/ros.h shim_ns/pcl/features/normal_3d.h normal_eigen.h

normal-port: libmcl3dl_normal_oracle.so

libmcl3dl_normal_oracle.so: normal_sampler_oracle.cpp normal_sampler_api.h normal_eigen.h ../include/mcl3dl_b200.h
	$(CXX) $(CXXFLAGS) -shared -o $@ normal_sampler_oracle.cpp

normal-ref: _ref/libmcl3dl_normal_ref.so

_ref/libmcl3dl_normal_ref.so: normal_sampler_ref_driver.cpp normal_sampler_api.h ../include/mcl3dl_b200.h $(SHIM_NS)
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -DPCL_NO_PRECOMPILE -Ishim_ns -Ishim -I$(REFERENCE)/include -shared -o $@ normal_sampler_ref_driver.cpp

normal-parity: _ref/normal_sampler_parity_test

_ref/normal_sampler_parity_test: normal_sampler_parity_test.cpp normal_sampler_oracle.cpp normal_sampler_api.h ../mcl_3dl_b200/host/lidar_measurement_model_b200.h ../include/mcl3dl_b200.h ../mcl_3dl_b200/libmcl3dl_b200.so $(SHIM_NS)
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -fPIE -DPCL_NO_PRECOMPILE -Ishim_ns -Ishim -I$(REFERENCE)/include -I../include -o $@ \
	    normal_sampler_parity_test.cpp normal_sampler_oracle.cpp $(REF_SOURCES) \
	    -L../mcl_3dl_b200 -lmcl3dl_b200 -Wl,-rpath,'$$ORIGIN/../../mcl_3dl_b200'

.PHONY: normal-port normal-ref normal-parity
