# Builds the mapping_skip_frame drivers of the reference's laserOdometry / laserMapping sources (test infrastructure) into
# oracle/_ref/, with the flags, paths and dependencies of Makefile (included): each driver includes the per-scan driver of the
# same node whole and adds its sequence / odometry-only entry points.  Only where /root/reference exists:
#   make -C oracle -f ref_skip.mk ref_skip
include Makefile
ref_skip: _ref/libref_odometry_seq.so _ref/libref_mapping_skip.so
_ref/libref_odometry_seq.so: ref_drivers/ref_odometry_seq.cc ref_drivers/ref_odometry.cc $(REF)/src/laserOdometry.cpp $(REF)/src/lidarFactor.hpp $(wildcard ref_shim/*/*) $(wildcard ref_shim/*/*/*) voxelgrid.cc kdtree.cc lm.cc oracle.h smallmath.h
	mkdir -p _ref
	$(CXX) $(REFFLAGS) -I $(REF)/src -DREF_LASER_ODOMETRY_CPP='"$(REF)/src/laserOdometry.cpp"' -shared -o $@ ref_drivers/ref_odometry_seq.cc voxelgrid.cc kdtree.cc lm.cc
_ref/libref_mapping_skip.so: ref_drivers/ref_mapping_skip.cc ref_drivers/ref_mapping.cc $(REF)/src/laserMapping.cpp $(REF)/src/lidarFactor.hpp $(wildcard ref_shim/*/*) $(wildcard ref_shim/*/*/*) voxelgrid.cc kdtree.cc lm.cc mapping.cc oracle.h smallmath.h
	mkdir -p _ref
	$(CXX) $(REFFLAGS) -I $(REF)/src -DREF_LASER_MAPPING_CPP='"$(REF)/src/laserMapping.cpp"' -shared -o $@ ref_drivers/ref_mapping_skip.cc voxelgrid.cc kdtree.cc lm.cc mapping.cc
.PHONY: ref_skip
