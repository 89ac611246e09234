# TEST INFRASTRUCTURE ONLY -- builds oracle/_ref/libref_box_search_{intended,o2}.so: the reference's getClusteredPoints and
# ruleBasedFilter over a C ABI (ref_box_search.cpp), the reference's side of box search's oracle (tests/box_search_scenes.py).
#
#   make -f box_search.mk   (after `make ref`: each helper links against the library whose functions it calls)
#
# The helper carries no copy of the reference: it is linked against libref_<mode>.so (rpath $ORIGIN), so the dynamic loader binds
# getClusteredPoints / ruleBasedFilter / sensorHeight to the instance already loaded by the test process.
REF      ?= /root/reference
OT       := $(REF)/object_tracking
OUT      := _ref
CXX      ?= g++
CXXFLAGS := -std=c++14 -O2 -w -fPIC
INC      := -I shim -I $(OT)/include -I $(OUT)/eigen_inc

.PHONY: all
all:
	@if [ -d "$(OT)" ]; then $(MAKE) --no-print-directory -f box_search.mk $(OUT)/libref_box_search_intended.so $(OUT)/libref_box_search_o2.so; \
	 else echo "oracle: $(REF) not present -- keeping prebuilt $(OUT)/libref_box_search_*.so"; fi

$(OUT)/libref_box_search_%.so: ref_box_search.cpp $(OUT)/libref_%.so
	$(CXX) $(CXXFLAGS) $(INC) -shared -o $@ ref_box_search.cpp -L $(OUT) -lref_$* -Wl,-rpath,'$$ORIGIN'
