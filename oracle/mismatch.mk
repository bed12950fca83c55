# oracle/mismatch.mk -- CHECKERS for the sparse-vector mismatch (test infrastructure, never the product).
#   liboracle_mismatch.so           the plain-C oracle plus orc_sv_mismatch / orc_sv_first_mismatch (bm_oracle_mismatch.c),
#                                   always buildable (gcc only)
#   _ref/libbmref_mismatch.so       the unmodified reference's sparse_vector_find_mismatch / sparse_vector_find_first_mismatch,
#                                   the closed forms through its bvector ops and a one-core timing entry (ref_mismatch_shim.cpp)
#   _ref/test_mismatch_binding      bm::b200::sparse_vector_find_mismatch / _first_mismatch against the reference
#   _ref/test_mismatch_binding64    the same harness under BM64ADDR (positions past 2^32)
# The last three need the reference tree; without it the tests use the recorded answers under tests/golden/ref.
REF ?= /root/reference/src
CC  ?= gcc
CXX ?= g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
ORACLE_SRCS := $(HERE)bm_oracle.c $(HERE)bm_oracle_entropy.c $(HERE)bm_synth.c $(HERE)bm_oracle_mismatch.c
BINDING_DEPS := $(HERE)test_mismatch_binding.cpp $(HERE)../bitmagic_b200/include/bmb200_aggregator.hpp $(HERE)../bitmagic_b200/include/bmb200_scanner.hpp $(HERE)../include/bmb200.h
BINDING_FLAGS := -std=c++17 -O2 -DBMAVX2OPT -march=skylake -mavx2 -pthread -I$(REF) -I$(HERE)../include -I$(HERE)../bitmagic_b200/include
BINDING_LIBS := -L$(HERE)../bitmagic_b200 -lbmb200 -Wl,-rpath,'$$ORIGIN/../../bitmagic_b200' -L/usr/local/cuda/lib64 -Wl,-rpath,/usr/local/cuda/lib64

all: $(HERE)liboracle_mismatch.so
	@if [ -d "$(REF)" ]; then $(MAKE) -f $(HERE)mismatch.mk $(HERE)_ref/libbmref_mismatch.so $(HERE)_ref/test_mismatch_binding \
	    $(HERE)_ref/test_mismatch_binding64; \
	else echo "oracle/mismatch.mk: $(REF) not present; using prebuilt oracle/_ref if any"; fi

$(HERE)liboracle_mismatch.so: $(ORACLE_SRCS) $(HERE)bm_oracle.h $(HERE)bm_oracle_int.h $(HERE)../include/bmb200.h
	$(CC) -O2 -std=c11 -fPIC -shared -Wall -pthread -o $@ $(ORACLE_SRCS)

$(HERE)_ref/libbmref_mismatch.so: $(HERE)ref_mismatch_shim.cpp
	mkdir -p $(HERE)_ref
	$(CXX) -std=c++17 -O2 -DBMAVX2OPT -march=skylake -mavx2 -fPIC -shared -pthread -I$(REF) -o $@ $(HERE)ref_mismatch_shim.cpp

$(HERE)_ref/test_mismatch_binding: $(BINDING_DEPS)
	mkdir -p $(HERE)_ref
	if [ -f $(HERE)../bitmagic_b200/libbmb200.so ]; then \
	$(CXX) $(BINDING_FLAGS) -o $@ $(HERE)test_mismatch_binding.cpp $(BINDING_LIBS); \
	else echo "libbmb200.so not built yet; skipping test_mismatch_binding"; fi

$(HERE)_ref/test_mismatch_binding64: $(BINDING_DEPS)
	mkdir -p $(HERE)_ref
	if [ -f $(HERE)../bitmagic_b200/libbmb200.so ]; then \
	$(CXX) $(BINDING_FLAGS) -DBM64ADDR -o $@ $(HERE)test_mismatch_binding.cpp $(BINDING_LIBS); \
	else echo "libbmb200.so not built yet; skipping test_mismatch_binding64"; fi

.PHONY: all
