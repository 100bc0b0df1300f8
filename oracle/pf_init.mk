# TEST INFRASTRUCTURE ONLY — the checkers of the resident set's initial seed, beside Makefile's (same compiler, flags and
# reference location, taken from it):
#   make -f pf_init.mk                 -> libmcl3dl_pf_init_oracle.so  (port; always buildable)
#   make -f pf_init.mk pf-init-ref     -> _ref/libmcl3dl_pf_init_ref.so (the reference's own initUsingNoiseGenerator,
#                                         generateNoise, setMean and MultivariateNoiseGenerator, header-only)
#   make -f pf_init.mk init-parity     -> _ref/init_parity_test (the configured start, cbPosition and a predict /
#                                         measure / resample cycle through the C++ adapter vs the reference filter; an
#                                         H100 runs it, tests/test_gpu_pf_init.py)
# The reference tier and the parity program compile against shim_mv/ first: MultivariateNoiseGenerator needs dynamic
# matrices and an eigensolver (repo-written stand-ins, not Eigen).
include Makefile
.DEFAULT_GOAL := pf-init-port

PFI_CXXFLAGS = $(CXXFLAGS) -Wno-subobject-linkage
REF_SOURCES = $(REFERENCE)/src/lidar_measurement_model_likelihood.cpp $(REFERENCE)/src/lidar_measurement_model_beam.cpp
SHIM_MV = shim_mv/Eigen/Core shim_mv/Eigen/Eigenvalues shim_mv/Eigen/LU shim_nd/Eigen/Core

pf-init-port: libmcl3dl_pf_init_oracle.so

libmcl3dl_pf_init_oracle.so: pf_init_oracle.cpp pf_init_api.h ../include/mcl3dl_b200.h
	$(CXX) $(PFI_CXXFLAGS) -shared -o $@ pf_init_oracle.cpp

pf-init-ref: _ref/libmcl3dl_pf_init_ref.so

_ref/libmcl3dl_pf_init_ref.so: pf_init_ref_driver.cpp pf_init_api.h ../include/mcl3dl_b200.h $(SHIM_MV)
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(PFI_CXXFLAGS) -Ishim_mv -Ishim -I$(REFERENCE)/include -shared -o $@ pf_init_ref_driver.cpp

init-parity: _ref/init_parity_test

_ref/init_parity_test: init_parity_test.cpp ../mcl_3dl_b200/host/lidar_measurement_model_b200.h ../include/mcl3dl_b200.h ../mcl_3dl_b200/libmcl3dl_b200.so $(SHIM_MV)
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -fPIE -DPCL_NO_PRECOMPILE -Ishim_mv -Ishim -I$(REFERENCE)/include -I../include -o $@ init_parity_test.cpp \
	    $(REF_SOURCES) -L../mcl_3dl_b200 -lmcl3dl_b200 -Wl,-rpath,'$$ORIGIN/../../mcl_3dl_b200'

.PHONY: pf-init-port pf-init-ref init-parity
