# TEST INFRASTRUCTURE ONLY — the checkers of global localisation and of the particle set's resize, beside Makefile's
# (same compiler, flags and reference location, taken from it):
#   make -f gl.mk              -> libmcl3dl_gl_oracle.so  (port; always buildable)
#   make -f gl.mk gl-ref       -> _ref/libmcl3dl_gl_ref.so (the reference's own ParticleFilter / Quat / State6DOF)
#   make -f gl.mk gl-parity    -> _ref/global_localization_parity_test (the service body and the node's shrink on the
#                                 reference filter vs the C++ adapter's resident calls; an H100 runs it,
#                                 tests/test_gpu_global_localization.py)
include Makefile
.DEFAULT_GOAL := gl-port

GL_CXXFLAGS = $(CXXFLAGS) -Wno-subobject-linkage
REF_SOURCES = $(REFERENCE)/src/lidar_measurement_model_likelihood.cpp $(REFERENCE)/src/lidar_measurement_model_beam.cpp

gl-port: libmcl3dl_gl_oracle.so

libmcl3dl_gl_oracle.so: gl_oracle.cpp gl_api.h ../include/mcl3dl_b200.h
	$(CXX) $(GL_CXXFLAGS) -shared -o $@ gl_oracle.cpp

gl-ref: _ref/libmcl3dl_gl_ref.so

_ref/libmcl3dl_gl_ref.so: gl_ref_driver.cpp ref_driver.cpp gl_api.h oracle_api.h ../include/mcl3dl_b200.h $(wildcard shim/*/*.h shim/*/*/*.h shim/Eigen/Core)
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(GL_CXXFLAGS) -DPCL_NO_PRECOMPILE -Ishim -I$(REFERENCE)/include -shared -o $@ gl_ref_driver.cpp $(REF_SOURCES)

gl-parity: _ref/global_localization_parity_test

_ref/global_localization_parity_test: global_localization_parity_test.cpp ../mcl_3dl_b200/host/lidar_measurement_model_b200.h ../include/mcl3dl_b200.h ../mcl_3dl_b200/libmcl3dl_b200.so
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -fPIE -DPCL_NO_PRECOMPILE -Ishim -I$(REFERENCE)/include -I../include -o $@ global_localization_parity_test.cpp \
	    $(REF_SOURCES) -L../mcl_3dl_b200 -lmcl3dl_b200 -Wl,-rpath,'$$ORIGIN/../../mcl_3dl_b200'

.PHONY: gl-port gl-ref gl-parity
