# Builds the MinMax search oracle (oracle/minmax_search.cpp, test infrastructure only) into liboracle_minmax_search.so,
# a library of its own next to liboracle.so, whose queue and distances it calls (build liboracle.so first).  Same flags
# as the main oracle.
# usage: make -C oracle -f minmax_search.mk
CXX ?= g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -mavx2 -mfma -mf16c -Wall -Wextra
liboracle_minmax_search.so: minmax_search.cpp oracle.h minmax_search.mk liboracle.so
	$(CXX) $(CXXFLAGS) -shared -o $@ minmax_search.cpp -L. -loracle -Wl,-rpath,'$$ORIGIN'
clean:
	rm -f liboracle_minmax_search.so
.PHONY: clean
