# Builds the filtered range search oracle (oracle/filtered_range_search.cpp, test infrastructure only) into liboracle_filtered_range_search.so,
# a library of its own next to liboracle.so, whose distances and queue it calls (build liboracle.so first).  Same flags
# as the main oracle.
# usage: make -C oracle -f filtered_range_search.mk
CXX ?= g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -mavx2 -mfma -mf16c -Wall -Wextra
liboracle_filtered_range_search.so: filtered_range_search.cpp oracle.h filtered_range_search.mk liboracle.so
	$(CXX) $(CXXFLAGS) -shared -o $@ filtered_range_search.cpp -L. -loracle -Wl,-rpath,'$$ORIGIN'
clean:
	rm -f liboracle_filtered_range_search.so
.PHONY: clean
