# init.mk — recipes of the start-of-sequence oracle pieces (TEST INFRASTRUCTURE ONLY), beside oracle/Makefile and with its flags:
#   make -f init.mk orc   liborc_init.so = orc_init.cpp (the restatement) over liborc.so; OUT=<dir> builds it elsewhere (a read-only tree)
#   make -f init.mk ref   _ref/libsdvref_init.so = ref_init_shim.cpp over _ref/libsdvref.so (the reference's own code, oracle/Makefile `ref`); only where the
#                         reference sources are present, like `ref`
CXX = /usr/bin/g++
CXXFLAGS = -std=c++17 -O3 -ffp-contract=off -fPIC -Wall -Wno-unused-variable
OUT ?= .
REF ?= /root/reference/src
REF_FLAGS = -std=c++14 -O3 -fPIC -ffp-contract=off -w -DNDEBUG -I ref_stub -I $(REF)
orc: $(OUT)/liborc_init.so
$(OUT)/liborc_init.so: orc_init.cpp liborc.so init.mk
	$(CXX) $(CXXFLAGS) -shared -o $@ orc_init.cpp -L. -lorc -Wl,-rpath,'$$ORIGIN' -Wl,-rpath,$(abspath .)
ref: _ref/libsdvref_init.so
_ref/libsdvref_init.so: ref_init_shim.cpp _ref/libsdvref.so init.mk $(wildcard ref_stub/*/*)
	$(CXX) $(REF_FLAGS) -shared -o $@ ref_init_shim.cpp -L_ref -lsdvref -Wl,-rpath,'$$ORIGIN'
.PHONY: orc ref
