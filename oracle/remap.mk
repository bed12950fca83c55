# oracle/remap.mk -- CHECKERS for the set image through a sparse vector (test infrastructure, never the product).
#   _ref/libbmref_remap.so        the unmodified reference's set2set_11_transform::remap behind a C wrapper, with a one-core
#                                 timing entry (ref_remap_shim.cpp), 32-bit addressing
#   _ref/libbmref_remap64.so      the same under BM64ADDR
#   _ref/test_remap_binding       bm::b200::set2set_11_transform against the reference
#   _ref/test_remap_binding64     the same harness under BM64ADDR
# All four need the reference tree; without it the tests use the recorded answers under tests/golden/ref.
REF ?= /root/reference/src
CXX ?= g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
SHIM_FLAGS := -std=c++17 -O2 -DBMAVX2OPT -march=skylake -mavx2 -fPIC -shared -pthread -I$(REF)
BINDING_DEPS := $(HERE)test_remap_binding.cpp $(HERE)../bitmagic_b200/include/bmb200_aggregator.hpp $(HERE)../bitmagic_b200/include/bmb200_scanner.hpp $(HERE)../include/bmb200.h
BINDING_FLAGS := -std=c++17 -O2 -DBMAVX2OPT -march=skylake -mavx2 -pthread -I$(REF) -I$(HERE)../include -I$(HERE)../bitmagic_b200/include
BINDING_LIBS := -L$(HERE)../bitmagic_b200 -lbmb200 -Wl,-rpath,'$$ORIGIN/../../bitmagic_b200' -L/usr/local/cuda/lib64 -Wl,-rpath,/usr/local/cuda/lib64

all:
	@if [ -d "$(REF)" ]; then $(MAKE) -f $(HERE)remap.mk $(HERE)_ref/libbmref_remap.so $(HERE)_ref/libbmref_remap64.so \
	    $(HERE)_ref/test_remap_binding $(HERE)_ref/test_remap_binding64; \
	else echo "oracle/remap.mk: $(REF) not present; using prebuilt oracle/_ref if any"; fi

$(HERE)_ref/libbmref_remap.so: $(HERE)ref_remap_shim.cpp
	mkdir -p $(HERE)_ref
	$(CXX) $(SHIM_FLAGS) -o $@ $(HERE)ref_remap_shim.cpp

$(HERE)_ref/libbmref_remap64.so: $(HERE)ref_remap_shim.cpp
	mkdir -p $(HERE)_ref
	$(CXX) $(SHIM_FLAGS) -DBM64ADDR -o $@ $(HERE)ref_remap_shim.cpp

$(HERE)_ref/test_remap_binding: $(BINDING_DEPS)
	mkdir -p $(HERE)_ref
	if [ -f $(HERE)../bitmagic_b200/libbmb200.so ]; then \
	$(CXX) $(BINDING_FLAGS) -o $@ $(HERE)test_remap_binding.cpp $(BINDING_LIBS); \
	else echo "libbmb200.so not built yet; skipping test_remap_binding"; fi

$(HERE)_ref/test_remap_binding64: $(BINDING_DEPS)
	mkdir -p $(HERE)_ref
	if [ -f $(HERE)../bitmagic_b200/libbmb200.so ]; then \
	$(CXX) $(BINDING_FLAGS) -DBM64ADDR -o $@ $(HERE)test_remap_binding.cpp $(BINDING_LIBS); \
	else echo "libbmb200.so not built yet; skipping test_remap_binding64"; fi

.PHONY: all
