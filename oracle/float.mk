# oracle/float.mk -- CHECKERS for the float scanner (test infrastructure, never the product).
#   liboracle_float.so        the plain-C oracle plus orc_scan_float (bm_oracle_float.c), always buildable (gcc only)
#   _ref/libbmref_float.so    the unmodified reference's sparse_vector_float and sparse_vector_scanner behind a C wrapper
#                             (ref_float_shim.cpp)
#   _ref/test_float_binding   bm::b200::scanner over sparse_vector_float against the reference
# The last two need the reference tree; without it the tests use the recorded answers under tests/golden/ref.
REF ?= /root/reference/src
CC  ?= gcc
CXX ?= g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
ORACLE_SRCS := $(HERE)bm_oracle.c $(HERE)bm_oracle_entropy.c $(HERE)bm_synth.c $(HERE)bm_oracle_float.c

all: $(HERE)liboracle_float.so
	@if [ -d "$(REF)" ]; then $(MAKE) -f $(HERE)float.mk $(HERE)_ref/libbmref_float.so $(HERE)_ref/test_float_binding; \
	else echo "oracle/float.mk: $(REF) not present; using prebuilt oracle/_ref if any"; fi

$(HERE)liboracle_float.so: $(ORACLE_SRCS) $(HERE)bm_oracle.h $(HERE)bm_oracle_int.h $(HERE)../include/bmb200.h
	$(CC) -O2 -std=c11 -fPIC -shared -Wall -pthread -o $@ $(ORACLE_SRCS)

$(HERE)_ref/libbmref_float.so: $(HERE)ref_float_shim.cpp $(HERE)../include/bmb200.h
	mkdir -p $(HERE)_ref
	$(CXX) -std=c++17 -O2 -DBMAVX2OPT -march=skylake -mavx2 -fPIC -shared -pthread -I$(REF) -o $@ $(HERE)ref_float_shim.cpp

$(HERE)_ref/test_float_binding: $(HERE)test_float_binding.cpp $(HERE)../bitmagic_b200/include/bmb200_aggregator.hpp $(HERE)../bitmagic_b200/include/bmb200_scanner.hpp $(HERE)../include/bmb200.h
	mkdir -p $(HERE)_ref
	if [ -f $(HERE)../bitmagic_b200/libbmb200.so ]; then \
	$(CXX) -std=c++17 -O2 -DBMAVX2OPT -march=skylake -mavx2 -pthread -I$(REF) -I$(HERE)../include -I$(HERE)../bitmagic_b200/include \
	    -o $@ $(HERE)test_float_binding.cpp -L$(HERE)../bitmagic_b200 -lbmb200 -Wl,-rpath,'$$ORIGIN/../../bitmagic_b200' -L/usr/local/cuda/lib64 -Wl,-rpath,/usr/local/cuda/lib64; \
	else echo "libbmb200.so not built yet; skipping test_float_binding"; fi

.PHONY: all
