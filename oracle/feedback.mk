# `make -C oracle -f feedback.mk` (after `make ref`): _ref/libviw_ref_feedback.so = refshim/ref_feedback_glue.cpp, entry points over the reference's
# own predictPtsInNextFrame / removeOutliers / setPrediction.  The reference's translation units are not compiled a second time: the glue
# links against _ref/libviw_ref.so, which holds them.  TEST INFRASTRUCTURE ONLY; _ref/ is git-ignored.
REF ?= $(VIWB_REFERENCE_DIR)/vins_estimator/src
CAM ?= $(VIWB_REFERENCE_DIR)/camera_models
_ref/libviw_ref_feedback.so: refshim/ref_feedback_glue.cpp _ref/libviw_ref.so refshim/mini_eigen.h refshim/mini_sophus.h refshim/ros_stub.h $(wildcard refshim/*/*.h*) $(wildcard refshim/*/*/*.h*)
	g++ -std=c++17 -O2 -fno-fast-math -ffp-contract=off -fPIC -w -fno-access-control -shared -I refshim -I $(REF) -I $(CAM)/include -o $@ refshim/ref_feedback_glue.cpp \
	    -L_ref -lviw_ref -Wl,-rpath,'$$ORIGIN' -lpthread
