# gamma.mk — recipes of the photometric-calibration oracle and pins (TEST INFRASTRUCTURE ONLY), beside oracle/Makefile and with its flags:
#   make -f gamma.mk orc   liborc_gamma.so = orc_gamma.cpp (makeImages' gamma weights) over liborc.so; OUT=<dir> builds it elsewhere (a read-only tree)
#   make -f gamma.mk ref   _ref/libsdvref_gamma.so = ref_gamma_shim.cpp over _ref/libsdvref.so (FullSystem::setGammaFunction, FrameHessian::makeImages with its CalibHessian)
#                          _ref/libsdvref_photo.so = the reference's Undistort.cpp + settings.cpp with ref_photo_shim.cpp's PGM reader in place of ImageRW_dummy.cpp
#                          (PhotometricUndistorter), self-contained and bound to its own symbols (-Bsymbolic): its settings are not libsdvref.so's;
#                          only where the reference sources are present, like oracle/Makefile `ref`
CXX = /usr/bin/g++
CXXFLAGS = -std=c++17 -O3 -ffp-contract=off -fPIC -Wall -Wno-unused-variable
OUT ?= .
REF ?= /root/reference/src
REF_FLAGS = -std=c++14 -O3 -fPIC -ffp-contract=off -w -DNDEBUG -I ref_stub -I $(REF)
orc: $(OUT)/liborc_gamma.so
$(OUT)/liborc_gamma.so: orc_gamma.cpp liborc.so gamma.mk
	$(CXX) $(CXXFLAGS) -shared -o $@ orc_gamma.cpp -L. -lorc -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,$(abspath .)
ref: _ref/libsdvref_gamma.so _ref/libsdvref_photo.so
_ref/libsdvref_gamma.so: ref_gamma_shim.cpp _ref/libsdvref.so gamma.mk $(wildcard ref_stub/*/*)
	$(CXX) $(REF_FLAGS) -shared -o $@ ref_gamma_shim.cpp -L_ref -lsdvref -Wl,-rpath,'$$ORIGIN'
_ref/libsdvref_photo.so: ref_photo_shim.cpp $(REF)/util/Undistort.cpp $(REF)/util/settings.cpp gamma.mk $(wildcard ref_stub/*/*) orc_math.hpp
	@mkdir -p _ref/photo
	$(CXX) $(REF_FLAGS) -c -o _ref/photo/Undistort.o $(REF)/util/Undistort.cpp
	$(CXX) $(REF_FLAGS) -c -o _ref/photo/settings.o $(REF)/util/settings.cpp
	$(CXX) $(REF_FLAGS) -shared -o $@ ref_photo_shim.cpp _ref/photo/Undistort.o _ref/photo/settings.o -Wl,-Bsymbolic -Wl,--no-undefined
.PHONY: orc ref
