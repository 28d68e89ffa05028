# Builds the transform oracle (oracle/transform.cpp, test infrastructure only) into liboracle_transform.so, a library of
# its own next to liboracle.so.  Same flags as the main oracle: every FMA is explicit (-ffp-contract=off) and the
# reference's default target is x86-64-v3; no -ffast-math, so subnormals are kept.
# usage: make -C oracle -f transform.mk
CXX ?= g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -mavx2 -mfma -mf16c -Wall -Wextra
liboracle_transform.so: transform.cpp transform.mk
	$(CXX) $(CXXFLAGS) -shared -o $@ transform.cpp
clean:
	rm -f liboracle_transform.so
.PHONY: clean
