# Builds the oracle of place recognition (test infrastructure, oracle/place.cc) into oracle/libplace.so, with the flags of
# Makefile (included; -ffp-contract=off):
#   make -C oracle -f place.mk libplace.so
include Makefile
libplace.so: place.cc
	$(CXX) $(CXXFLAGS) -shared -o $@ place.cc
