# oracle/in.mk -- CHECKERS for the set-membership search (test infrastructure, never the product).
#   liboracle_in.so       the plain-C oracle plus orc_scan_in (bm_oracle_in.c), always buildable (gcc only)
#   _ref/libbmref_in.so   the unmodified reference's iterator find_eq over sparse_vector<> / rsc_sparse_vector<> behind a C
#                         wrapper (ref_in_shim.cpp)
#   _ref/test_in_binding  bm::b200::scanner's find_eq(first, last, bv_out) / count_eq against the reference
# The last two need the reference tree; without it the tests use the recorded answers under tests/golden/ref.
REF ?= /root/reference/src
CC  ?= gcc
CXX ?= g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
ORACLE_SRCS := $(HERE)bm_oracle.c $(HERE)bm_oracle_entropy.c $(HERE)bm_synth.c $(HERE)bm_oracle_in.c

all: $(HERE)liboracle_in.so
	@if [ -d "$(REF)" ]; then $(MAKE) -f $(HERE)in.mk $(HERE)_ref/libbmref_in.so $(HERE)_ref/test_in_binding; \
	else echo "oracle/in.mk: $(REF) not present; using prebuilt oracle/_ref if any"; fi

$(HERE)liboracle_in.so: $(ORACLE_SRCS) $(HERE)bm_oracle.h $(HERE)bm_oracle_int.h $(HERE)../include/bmb200.h
	$(CC) -O2 -std=c11 -fPIC -shared -Wall -pthread -o $@ $(ORACLE_SRCS)

$(HERE)_ref/libbmref_in.so: $(HERE)ref_in_shim.cpp $(HERE)../include/bmb200.h
	mkdir -p $(HERE)_ref
	$(CXX) -std=c++17 -O2 -DBMAVX2OPT -march=skylake -mavx2 -fPIC -shared -pthread -I$(REF) -o $@ $(HERE)ref_in_shim.cpp

$(HERE)_ref/test_in_binding: $(HERE)test_in_binding.cpp $(HERE)../bitmagic_b200/include/bmb200_aggregator.hpp $(HERE)../bitmagic_b200/include/bmb200_scanner.hpp $(HERE)../include/bmb200.h
	mkdir -p $(HERE)_ref
	if [ -f $(HERE)../bitmagic_b200/libbmb200.so ]; then \
	$(CXX) -std=c++17 -O2 -DBMAVX2OPT -march=skylake -mavx2 -pthread -I$(REF) -I$(HERE)../include -I$(HERE)../bitmagic_b200/include \
	    -o $@ $(HERE)test_in_binding.cpp -L$(HERE)../bitmagic_b200 -lbmb200 -Wl,-rpath,'$$ORIGIN/../../bitmagic_b200' -L/usr/local/cuda/lib64 -Wl,-rpath,/usr/local/cuda/lib64; \
	else echo "libbmb200.so not built yet; skipping test_in_binding"; fi

.PHONY: all
