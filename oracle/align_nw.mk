# ORACLE / TEST INFRASTRUCTURE ONLY: the checkers of mashmap-b200 --align, edlib's global (NW) mode
# (make -f oracle/align_nw.mk).
#   libalign_nw_oracle.so    full-matrix CPU restatement of edlib's NW/PATH decisions (align_nw_oracle.cpp); travels alone
#   _ref/libedlib_nw_ref.so  edlibAlign(NW, PATH) of the reference's header-only edlib, callable per pair (edlib_nw_harness.cpp)
# The _ref target is built only where the reference's sources are readable; nothing from it enters git.
REF ?= /root/reference
CXX := /usr/bin/g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

all: oracle ref

oracle: $(HERE)libalign_nw_oracle.so

$(HERE)libalign_nw_oracle.so: $(HERE)align_nw_oracle.cpp $(HERE)align_oracle.cpp
	$(CXX) -O2 -std=c++17 -Wall -fPIC -shared -fvisibility=hidden $< -o $@

ref:
	@if [ -d $(REF)/src/common ]; then $(MAKE) -f $(HERE)align_nw.mk $(HERE)_ref/libedlib_nw_ref.so; \
	 else echo "[oracle] $(REF) not present: keeping prebuilt oracle/_ref"; fi

$(HERE)_ref/libedlib_nw_ref.so: $(HERE)edlib_nw_harness.cpp $(HERE)edlib_harness.cpp
	@mkdir -p $(HERE)_ref
	$(CXX) -O2 -std=c++17 -w -fPIC -shared -fvisibility=hidden -I$(REF)/src/common $< -o $@

clean:
	rm -rf $(HERE)_ref/libedlib_nw_ref.so $(HERE)libalign_nw_oracle.so
