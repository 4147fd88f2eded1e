# `make -C oracle -f features.mk` (after `make ref`): _ref/libviw_ref_features.so = refshim/ref_features_glue.cpp, entry points that drive the
# reference's own FeatureManager.  feature_manager.cpp is not compiled a second time: the glue links against _ref/libviw_ref.so, which holds it.
# TEST INFRASTRUCTURE ONLY; _ref/ is git-ignored.
REF ?= $(VIWB_REFERENCE_DIR)/vins_estimator/src
CAM ?= $(VIWB_REFERENCE_DIR)/camera_models
_ref/libviw_ref_features.so: refshim/ref_features_glue.cpp _ref/libviw_ref.so refshim/mini_eigen.h refshim/mini_sophus.h refshim/ros_stub.h $(wildcard refshim/*/*.h*) $(wildcard refshim/*/*/*.h*)
	g++ -std=c++17 -O2 -fno-fast-math -ffp-contract=off -fPIC -w -fno-access-control -shared -I refshim -I $(REF) -I $(CAM)/include -o $@ refshim/ref_features_glue.cpp \
	    -L_ref -lviw_ref -Wl,-rpath,'$$ORIGIN' -lpthread
