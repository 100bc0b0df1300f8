# TEST INFRASTRUCTURE ONLY — the checkers of the matched / unmatched output, beside Makefile's (same compiler, flags and
# reference location, taken from it):
#   make -f match.mk              -> libmcl3dl_match_oracle.so  (port; always buildable)
#   make -f match.mk match-ref    -> _ref/libmcl3dl_match_ref.so (the reference's own loop, sources where they lie)
#   make -f match.mk match-parity -> _ref/match_parity_test      (reference loop vs the C++ adapter's matchOutput; an
#                                    H100 runs it, tests/test_gpu_match_output.py)
include Makefile
.DEFAULT_GOAL := match-port

# the two sources include whole checker files, whose internal types then sit in a struct with external linkage
MATCH_CXXFLAGS = $(CXXFLAGS) -Wno-subobject-linkage
REF_SOURCES = $(REFERENCE)/src/lidar_measurement_model_likelihood.cpp $(REFERENCE)/src/lidar_measurement_model_beam.cpp

match-port: libmcl3dl_match_oracle.so

libmcl3dl_match_oracle.so: match_oracle.cpp mcl3dl_oracle.cpp match_api.h oracle_api.h ../include/mcl3dl_b200.h
	$(CXX) $(MATCH_CXXFLAGS) -shared -o $@ match_oracle.cpp

match-ref: _ref/libmcl3dl_match_ref.so

_ref/libmcl3dl_match_ref.so: match_ref_driver.cpp ref_driver.cpp match_api.h oracle_api.h ../include/mcl3dl_b200.h $(wildcard shim/*/*.h shim/*/*/*.h shim/Eigen/Core)
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(MATCH_CXXFLAGS) -DPCL_NO_PRECOMPILE -Ishim -I$(REFERENCE)/include -shared -o $@ match_ref_driver.cpp $(REF_SOURCES)

match-parity: _ref/match_parity_test

_ref/match_parity_test: match_parity_test.cpp ../mcl_3dl_b200/host/lidar_measurement_model_b200.h ../include/mcl3dl_b200.h ../mcl_3dl_b200/libmcl3dl_b200.so
	@test -d $(REFERENCE)/include/mcl_3dl || (echo "reference tree not present at $(REFERENCE)"; exit 1)
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -fPIE -DPCL_NO_PRECOMPILE -Ishim -I$(REFERENCE)/include -I../include -o $@ match_parity_test.cpp \
	    $(REF_SOURCES) -L../mcl_3dl_b200 -lmcl3dl_b200 -Wl,-rpath,'$$ORIGIN/../../mcl_3dl_b200'

.PHONY: match-port match-ref match-parity
