# Builds the table-distance range search oracle (oracle/range_table.cpp, test infrastructure only) into
# liboracle_range_table.so, a library of its own next to liboracle.so, whose queue and distances it calls (build
# liboracle.so first).  Same flags as the main oracle.
# usage: make -C oracle -f range_table.mk
CXX ?= g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -mavx2 -mfma -mf16c -Wall -Wextra
liboracle_range_table.so: range_table.cpp oracle.h range_table.mk liboracle.so
	$(CXX) $(CXXFLAGS) -shared -o $@ range_table.cpp -L. -loracle -Wl,-rpath,'$$ORIGIN'
clean:
	rm -f liboracle_range_table.so
.PHONY: clean
