# Builds the oracle's published-cloud restatements (test infrastructure, oracle/clouds.cc) into oracle/libclouds.so, with the flags
# of Makefile (included):
#   make -C oracle -f clouds.mk libclouds.so
include Makefile
libclouds.so: clouds.cc oracle.h smallmath.h
	$(CXX) $(CXXFLAGS) -shared -o $@ clouds.cc
