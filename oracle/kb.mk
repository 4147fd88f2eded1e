# `make -C oracle -f kb.mk`: libvo_kb.so = vo_kb.c, the restated Kannala-Brandt lift / projection and Eigen 3.3's nonsymmetric eigen-solver,
# compiled with -ffp-contract=off so that no product is fused and the trigonometric functions are glibc's.
# `make -C oracle -f kb.mk ref` (after `make ref`): _ref/libviw_ref_kb.so = the reference's camera_models/src/camera_models/EquidistantCamera.cc
# compiled unmodified, with refshim/ref_kb_glue.cpp (entry points over FeatureTracker::undistortedPts and spaceToPlane with an
# EquidistantCamera) and vo_kb.c, whose eigen-solver stands in for Eigen's EigenSolver (refshim/kb_shim.h, forced in with cv_svd.h: the
# EigenSolver and the Point2d-from-Point2f conversion the file needs beyond the stand-ins of refshim/).  Linked against
# _ref/libviw_ref.so, which holds FeatureTracker, Camera.cc and PinholeCamera.cc.  The names still undefined after a first link (the
# calibration routines: estimateIntrinsics' helpers, cv::SVD::solveZ, initUndistort*'s cv::convertMaps, ...) become refshim/gen_stubs.py's
# aborting stubs, as in camera.mk.  TEST INFRASTRUCTURE ONLY; _ref/ is git-ignored.
REF ?= $(VIWB_REFERENCE_DIR)/vins_estimator/src
CAM ?= $(VIWB_REFERENCE_DIR)/camera_models
KBFLAGS = -O2 -fPIC -fno-fast-math -ffp-contract=off
CXXFLAGS = -std=c++17 $(KBFLAGS) -w -I refshim -I $(REF) -I $(CAM)/include
LINK = -L_ref -lviw_ref -Wl,-rpath,'$$ORIGIN' -lpthread
libvo_kb.so: vo_kb.c
	gcc -std=c11 $(KBFLAGS) -Wall -shared -o $@ vo_kb.c -lm
ref: _ref/libviw_ref_kb.so
_ref/libviw_ref_kb.so: refshim/ref_kb_glue.cpp refshim/cv_svd.h refshim/kb_shim.h refshim/gen_stubs.py vo_kb.c _ref/libviw_ref.so $(CAM)/src/camera_models/EquidistantCamera.cc refshim/mini_eigen.h refshim/ros_stub.h $(wildcard refshim/*/*.h*) $(wildcard refshim/*/*/*.h*)
	g++ $(CXXFLAGS) -include refshim/cv_svd.h -include refshim/kb_shim.h -c -o _ref/EquidistantCamera.o $(CAM)/src/camera_models/EquidistantCamera.cc
	g++ $(CXXFLAGS) -fno-access-control -c -o _ref/ref_kb_glue.o refshim/ref_kb_glue.cpp
	gcc -std=c11 $(KBFLAGS) -c -o _ref/vo_kb_ref.o vo_kb.c
	g++ -shared -o _ref/pass1k.so _ref/ref_kb_glue.o _ref/EquidistantCamera.o _ref/vo_kb_ref.o $(LINK) -lm
	python3 refshim/gen_stubs.py _ref/pass1k.so _ref/ref_stubs_k_all.c
	nm -D --defined-only _ref/libviw_ref.so | awk '{print " " $$3 "("}' > _ref/ref_defined_k.txt
	grep -v -F -f _ref/ref_defined_k.txt _ref/ref_stubs_k_all.c > _ref/ref_stubs_k.c
	gcc -O1 -fPIC -w -c -o _ref/ref_stubs_k.o _ref/ref_stubs_k.c
	g++ -shared -o $@ _ref/ref_kb_glue.o _ref/EquidistantCamera.o _ref/vo_kb_ref.o _ref/ref_stubs_k.o $(LINK) -lm
	rm -f _ref/pass1k.so
