# Builds the in-place delete oracle (oracle/inplace_delete.cpp, test infrastructure only) into
# liboracle_inplace_delete.so, a library of its own next to liboracle.so, whose distances, queue and prune it calls
# (build liboracle.so first).  Same flags as the main oracle.
# usage: make -C oracle -f inplace_delete.mk
CXX ?= g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -mavx2 -mfma -mf16c -Wall -Wextra
liboracle_inplace_delete.so: inplace_delete.cpp oracle.h inplace_delete.mk liboracle.so
	$(CXX) $(CXXFLAGS) -shared -o $@ inplace_delete.cpp -L. -loracle -Wl,-rpath,'$$ORIGIN'
clean:
	rm -f liboracle_inplace_delete.so
.PHONY: clean
