# Builds the table-distance diverse search oracle (oracle/diverse_table.cpp, test infrastructure only) into
# liboracle_diverse_table.so, linked against liboracle_diverse_search.so, whose DiverseNeighborQueue it drives, and
# liboracle.so, whose distances the rerank calls (build both first).  Same flags as the main oracle.
# usage: make -C oracle -f diverse_table.mk
CXX ?= g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -ffp-contract=off -fno-fast-math -mavx2 -mfma -mf16c -Wall -Wextra
liboracle_diverse_table.so: diverse_table.cpp oracle.h diverse_table.mk liboracle.so liboracle_diverse_search.so
	$(CXX) $(CXXFLAGS) -shared -o $@ diverse_table.cpp -L. -loracle_diverse_search -loracle -Wl,-rpath,'$$ORIGIN'
clean:
	rm -f liboracle_diverse_table.so
.PHONY: clean
