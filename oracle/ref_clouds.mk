# Builds the published-cloud driver of the reference's laserMapping source (test infrastructure) into oracle/_ref/, with the
# flags, paths and dependencies of Makefile (included): ref_mapping_clouds.cc includes the per-frame mapping driver whole and
# adds read-back of /laser_cloud_surround, /laser_cloud_map and /velodyne_cloud_registered.  Only where /root/reference exists:
#   make -C oracle -f ref_clouds.mk ref_clouds
include Makefile
ref_clouds: _ref/libref_mapping_clouds.so
_ref/libref_mapping_clouds.so: ref_drivers/ref_mapping_clouds.cc ref_drivers/ref_mapping.cc $(REF)/src/laserMapping.cpp $(REF)/src/lidarFactor.hpp $(wildcard ref_shim/*/*) $(wildcard ref_shim/*/*/*) voxelgrid.cc kdtree.cc lm.cc mapping.cc oracle.h smallmath.h
	mkdir -p _ref
	$(CXX) $(REFFLAGS) -I $(REF)/src -DREF_LASER_MAPPING_CPP='"$(REF)/src/laserMapping.cpp"' -shared -o $@ ref_drivers/ref_mapping_clouds.cc voxelgrid.cc kdtree.cc lm.cc mapping.cc
.PHONY: ref_clouds
