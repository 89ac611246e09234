# TEST INFRASTRUCTURE ONLY -- builds oracle/_ref/libref_retire_{intended,tunable}.so: ref_tracker_retire (ref_retire.cpp) on the
# track table of libref_intended.so / libref_tunable.so, the oracle of track retirement (oracle/ref_retire.py).
#
#   make -f retire.mk   (after `make ref` and `make -f tunable.mk`: each helper links against the library whose table it erases)
#
# The helper carries no copy of the reference: it is linked against libref_<mode>.so (rpath $ORIGIN), so the dynamic loader binds
# its targets_ / trackNumVec_ to the instance already loaded by the test process.
REF      ?= /root/reference
OT       := $(REF)/object_tracking
OUT      := _ref
CXX      ?= g++
CXXFLAGS := -std=c++14 -O2 -w -fPIC
INC      := -I shim -I $(OT)/include -I $(OUT)/eigen_inc

.PHONY: all
all:
	@if [ -d "$(OT)" ]; then $(MAKE) --no-print-directory -f retire.mk $(OUT)/libref_retire_intended.so $(OUT)/libref_retire_tunable.so; \
	 else echo "oracle: $(REF) not present -- keeping prebuilt $(OUT)/libref_retire_*.so"; fi

$(OUT)/libref_retire_%.so: ref_retire.cpp $(OUT)/libref_%.so
	$(CXX) $(CXXFLAGS) $(INC) -shared -o $@ ref_retire.cpp -L $(OUT) -lref_$* -Wl,-rpath,'$$ORIGIN'
