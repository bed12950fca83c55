# oracle/str.mk -- CHECKERS for the string scanner (test infrastructure, never the product).
#   liboracle_str.so       the plain-C oracle plus orc_scan_str (bm_oracle_str.c), always buildable (gcc only)
#   _ref/libbmref_str.so   the unmodified reference's str_sparse_vector and sparse_vector_scanner behind a C wrapper
#                          (ref_str_shim.cpp)
#   _ref/test_str_binding  bm::b200::scanner over str_sparse_vector against the reference
# The last two need the reference tree; without it the tests use the recorded answers under tests/golden/ref.
REF ?= /root/reference/src
CC  ?= gcc
CXX ?= g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
ORACLE_SRCS := $(HERE)bm_oracle.c $(HERE)bm_oracle_entropy.c $(HERE)bm_synth.c $(HERE)bm_oracle_str.c

all: $(HERE)liboracle_str.so
	@if [ -d "$(REF)" ]; then $(MAKE) -f $(HERE)str.mk $(HERE)_ref/libbmref_str.so $(HERE)_ref/test_str_binding; \
	else echo "oracle/str.mk: $(REF) not present; using prebuilt oracle/_ref if any"; fi

$(HERE)liboracle_str.so: $(ORACLE_SRCS) $(HERE)bm_oracle.h $(HERE)bm_oracle_int.h $(HERE)../include/bmb200.h
	$(CC) -O2 -std=c11 -fPIC -shared -Wall -pthread -o $@ $(ORACLE_SRCS)

$(HERE)_ref/libbmref_str.so: $(HERE)ref_str_shim.cpp $(HERE)../include/bmb200.h
	mkdir -p $(HERE)_ref
	$(CXX) -std=c++17 -O2 -DBMAVX2OPT -march=skylake -mavx2 -fPIC -shared -pthread -I$(REF) -o $@ $(HERE)ref_str_shim.cpp

$(HERE)_ref/test_str_binding: $(HERE)test_str_binding.cpp $(HERE)../bitmagic_b200/include/bmb200_aggregator.hpp $(HERE)../bitmagic_b200/include/bmb200_scanner.hpp $(HERE)../include/bmb200.h
	mkdir -p $(HERE)_ref
	if [ -f $(HERE)../bitmagic_b200/libbmb200.so ]; then \
	$(CXX) -std=c++17 -O2 -DBMAVX2OPT -march=skylake -mavx2 -pthread -I$(REF) -I$(HERE)../include -I$(HERE)../bitmagic_b200/include \
	    -o $@ $(HERE)test_str_binding.cpp -L$(HERE)../bitmagic_b200 -lbmb200 -Wl,-rpath,'$$ORIGIN/../../bitmagic_b200' -L/usr/local/cuda/lib64 -Wl,-rpath,/usr/local/cuda/lib64; \
	else echo "libbmb200.so not built yet; skipping test_str_binding"; fi

.PHONY: all
