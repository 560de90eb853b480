# ORACLE / TEST INFRASTRUCTURE ONLY: the static-band restatement of edlib's global (NW) mode (make -f oracle/align_band.mk).
#   libalign_band_oracle.so  align_nw_oracle.cpp's rules with every banded sweep restricted to the band (align_band_oracle.cpp)
CXX := /usr/bin/g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

all: $(HERE)libalign_band_oracle.so

$(HERE)libalign_band_oracle.so: $(HERE)align_band_oracle.cpp $(HERE)align_oracle.cpp
	$(CXX) -O2 -std=c++17 -Wall -fPIC -shared -fvisibility=hidden $< -o $@

clean:
	rm -f $(HERE)libalign_band_oracle.so
