# `make -C oracle -f camera.mk` (after `make ref`): _ref/libviw_ref_camera.so = the reference's camera_models/src/camera_models/CataCamera.cc
# (the MEI model), compiled unmodified, and refshim/ref_camera_glue.cpp, entry points over it and over the FeatureTracker members that call a
# camera.  The reference's other translation units are not compiled a second time: the library links against _ref/libviw_ref.so, which
# holds them.  CataCamera.cc names cv::SVD::solveZ, which the OpenCV stand-ins lack: refshim/cv_svd.h declares it, forced in with -include.
# Two-pass link as in the Makefile's `ref` recipe: the names still undefined after a first link that libviw_ref.so does not define either
# become refshim/gen_stubs.py's aborting stubs.  TEST INFRASTRUCTURE ONLY; _ref/ is git-ignored.
REF ?= $(VIWB_REFERENCE_DIR)/vins_estimator/src
CAM ?= $(VIWB_REFERENCE_DIR)/camera_models
CXXFLAGS = -std=c++17 -O2 -fno-fast-math -ffp-contract=off -fPIC -w -I refshim -I $(REF) -I $(CAM)/include
LINK = -L_ref -lviw_ref -Wl,-rpath,'$$ORIGIN' -lpthread
_ref/libviw_ref_camera.so: refshim/ref_camera_glue.cpp refshim/cv_svd.h refshim/gen_stubs.py _ref/libviw_ref.so $(CAM)/src/camera_models/CataCamera.cc refshim/mini_eigen.h refshim/ros_stub.h $(wildcard refshim/*/*.h*) $(wildcard refshim/*/*/*.h*)
	g++ $(CXXFLAGS) -include refshim/cv_svd.h -c -o _ref/CataCamera.o $(CAM)/src/camera_models/CataCamera.cc
	g++ $(CXXFLAGS) -fno-access-control -c -o _ref/ref_camera_glue.o refshim/ref_camera_glue.cpp
	g++ -shared -o _ref/pass1c.so _ref/ref_camera_glue.o _ref/CataCamera.o $(LINK)
	python3 refshim/gen_stubs.py _ref/pass1c.so _ref/ref_stubs_c_all.c
	nm -D --defined-only _ref/libviw_ref.so | awk '{print " " $$3 "("}' > _ref/ref_defined.txt
	grep -v -F -f _ref/ref_defined.txt _ref/ref_stubs_c_all.c > _ref/ref_stubs_c.c
	gcc -O1 -fPIC -w -c -o _ref/ref_stubs_c.o _ref/ref_stubs_c.c
	g++ -shared -o $@ _ref/ref_camera_glue.o _ref/CataCamera.o _ref/ref_stubs_c.o $(LINK)
	rm -f _ref/pass1c.so
