# TEST INFRASTRUCTURE ONLY — the checkers of the ray markers (mcl3dl_beam_cast), beside Makefile's (same compiler, flags
# and reference location, taken from it):
#   make -f beam_cast.mk                  -> libmcl3dl_beam_cast_oracle.so  (port; always buildable)
#   make -f beam_cast.mk beam-cast-ref    -> _ref/libmcl3dl_beam_cast_ref.so (the node's marker loop on the reference's
#                                            own beam model, sources where they lie)
#   make -f beam_cast.mk beam-cast-parity -> _ref/beam_cast_parity_test      (that loop vs the C++ adapter's castBeams,
#                                            and a node without its CPU map index; an H100 runs it,
#                                            tests/test_gpu_beam_cast.py)
include Makefile
.DEFAULT_GOAL := beam-cast-port

# the two sources include whole checker files, whose internal types then sit in a struct with external linkage
BEAM_CAST_CXXFLAGS = $(CXXFLAGS) -Wno-subobject-linkage
REF_SOURCES = $(REFERENCE)/src/lidar_measurement_model_likelihood.cpp $(REFERENCE)/src/lidar_measurement_model_beam.cpp

beam-cast-port: libmcl3dl_beam_cast_oracle.so

libmcl3dl_beam_cast_oracle.so: beam_cast_oracle.cpp mcl3dl_oracle.cpp beam_cast_api.h oracle_api.h ../include/mcl3dl_b200.h
	$(CXX) $(BEAM_CAST_CXXFLAGS) -shared -o $@ beam_cast_oracle.cpp

beam-cast-ref: _ref/libmcl3dl_beam_cast_ref.so

_ref/libmcl3dl_beam_cast_ref.so: beam_cast_ref_driver.cpp ref_driver.cpp beam_cast_api.h oracle_api.h ../include/mcl3dl_b200.h $(wildcard shim/*/*.h shim/*/*/*.h shim/Eigen/Core)
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(BEAM_CAST_CXXFLAGS) -DPCL_NO_PRECOMPILE -Ishim -I$(REFERENCE)/include -shared -o $@ beam_cast_ref_driver.cpp $(REF_SOURCES)

beam-cast-parity: _ref/beam_cast_parity_test

_ref/beam_cast_parity_test: beam_cast_parity_test.cpp ../mcl_3dl_b200/host/lidar_measurement_model_b200.h ../include/mcl3dl_b200.h ../mcl_3dl_b200/libmcl3dl_b200.so
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -fPIE -DPCL_NO_PRECOMPILE -Ishim -I$(REFERENCE)/include -I../include -o $@ beam_cast_parity_test.cpp \
	    $(REF_SOURCES) -L../mcl_3dl_b200 -lmcl3dl_b200 -Wl,-rpath,'$$ORIGIN/../../mcl_3dl_b200'

.PHONY: beam-cast-port beam-cast-ref beam-cast-parity
