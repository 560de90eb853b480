# ORACLE / TEST INFRASTRUCTURE ONLY: the checkers of mashmap-b200-align (make -f oracle/align.mk).
#   libalign_oracle.so      full-matrix CPU restatement of edlib's HW/PATH decisions (align_oracle.cpp); travels alone
#   _ref/mashmap_align_ref  the UNMODIFIED reference aligner (src/align/align.cpp), compiled like _ref/mashmap_ref
#   _ref/libedlib_ref.so    edlibAlign(HW, PATH) of the reference's header-only edlib, callable per pair (edlib_harness.cpp)
# The _ref targets are built only where the reference's sources are readable; nothing from them enters git.
REF ?= /root/reference
CXX := /usr/bin/g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REFINC := -I$(REF)/src -I$(REF)/src/common -I$(HERE)gsl_shim -I$(HERE)
OPT := -O3 -std=c++17 -w

all: oracle ref

oracle: $(HERE)libalign_oracle.so

$(HERE)libalign_oracle.so: $(HERE)align_oracle.cpp
	$(CXX) -O2 -std=c++17 -Wall -fPIC -shared -fvisibility=hidden $< -o $@

ref:
	@if [ -d $(REF)/src/align ]; then $(MAKE) -f $(HERE)align.mk $(HERE)_ref/mashmap_align_ref $(HERE)_ref/libedlib_ref.so; \
	 else echo "[oracle] $(REF) not present: keeping prebuilt oracle/_ref"; fi

$(HERE)_ref/mashmap_align_ref: $(REF)/src/align/align.cpp $(HERE)gsl_shim/gsl/gsl_cdf.h
	@mkdir -p $(HERE)_ref
	$(CXX) $(OPT) $(REFINC) $(REF)/src/common/utils.cpp $(REF)/src/align/align.cpp -o $@ -lz -lpthread

$(HERE)_ref/libedlib_ref.so: $(HERE)edlib_harness.cpp
	@mkdir -p $(HERE)_ref
	$(CXX) -O2 -std=c++17 -w -fPIC -shared -fvisibility=hidden -I$(REF)/src/common $< -o $@

clean:
	rm -rf $(HERE)_ref/mashmap_align_ref $(HERE)_ref/libedlib_ref.so $(HERE)libalign_oracle.so
