# Builds the insert oracle (oracle/insert.cpp, test infrastructure only) into liboracle_insert.so, a library of its own
# next to liboracle.so, whose distances, queue and prune it calls (build liboracle.so first).  Same flags as the main
# oracle.
# usage: make -C oracle -f insert.mk
CXX ?= g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -mavx2 -mfma -mf16c -Wall -Wextra
liboracle_insert.so: insert.cpp oracle.h insert.mk liboracle.so
	$(CXX) $(CXXFLAGS) -shared -o $@ insert.cpp -L. -loracle -Wl,-rpath,'$$ORIGIN'
clean:
	rm -f liboracle_insert.so
.PHONY: clean
