# Builds the oracle's frozen-map frame (test infrastructure, oracle/frozen.cc: localisation against a prior map) into
# oracle/libfrozen.so, with the flags of Makefile (included):
#   make -C oracle -f frozen.mk libfrozen.so
include Makefile
libfrozen.so: frozen.cc voxelgrid.cc kdtree.cc lm.cc mapping.cc oracle.h smallmath.h
	$(CXX) $(CXXFLAGS) -shared -o $@ frozen.cc voxelgrid.cc kdtree.cc lm.cc mapping.cc
