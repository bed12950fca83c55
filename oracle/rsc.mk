# oracle/rsc.mk -- CHECKERS for the rank-select compressed sparse vector path (test infrastructure, never the product).
#   _ref/libbmref_rsc.so    the unmodified reference's rsc_sparse_vector / sparse_vector_scanner / rank_compressor
#                           behind a C wrapper (ref_rsc_shim.cpp)
#   _ref/test_rsc_binding   bm::b200::scanner<rsc_sparse_vector> and bm::b200::rank_compressor against the reference
# Both need the reference tree; without it nothing is built and the tests use the recorded answers under tests/golden/ref.
REF ?= /root/reference/src
CXX ?= g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

all:
	@if [ -d "$(REF)" ]; then $(MAKE) -f $(HERE)rsc.mk $(HERE)_ref/libbmref_rsc.so $(HERE)_ref/test_rsc_binding; \
	else echo "oracle/rsc.mk: $(REF) not present; using prebuilt oracle/_ref if any"; fi

$(HERE)_ref/libbmref_rsc.so: $(HERE)ref_rsc_shim.cpp $(HERE)../include/bmb200.h
	mkdir -p $(HERE)_ref
	$(CXX) -std=c++17 -O2 -DBMAVX2OPT -march=skylake -mavx2 -fPIC -shared -pthread -I$(REF) -o $@ $(HERE)ref_rsc_shim.cpp

$(HERE)_ref/test_rsc_binding: $(HERE)test_rsc_binding.cpp $(HERE)../bitmagic_b200/include/bmb200_aggregator.hpp $(HERE)../bitmagic_b200/include/bmb200_scanner.hpp $(HERE)../include/bmb200.h
	mkdir -p $(HERE)_ref
	if [ -f $(HERE)../bitmagic_b200/libbmb200.so ]; then \
	$(CXX) -std=c++17 -O2 -DBMAVX2OPT -march=skylake -mavx2 -pthread -I$(REF) -I$(HERE)../include -I$(HERE)../bitmagic_b200/include \
	    -o $@ $(HERE)test_rsc_binding.cpp -L$(HERE)../bitmagic_b200 -lbmb200 -Wl,-rpath,'$$ORIGIN/../../bitmagic_b200' -L/usr/local/cuda/lib64 -Wl,-rpath,/usr/local/cuda/lib64; \
	else echo "libbmb200.so not built yet; skipping test_rsc_binding"; fi

.PHONY: all
