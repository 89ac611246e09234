# TEST INFRASTRUCTURE ONLY -- builds oracle/_ref/libref_predict_{intended,tunable}.so: ref_tracker_predict (ref_predict.cpp) on the
# track table of libref_intended.so / libref_tunable.so, the oracle of track prediction (oracle/ref_predict.py).
#
#   make -f predict.mk   (after `make ref` and `make -f tunable.mk`: each helper links against the library whose table it reads)
#
# The helper carries no copy of the reference: it is linked against libref_<mode>.so (rpath $ORIGIN), so the dynamic loader binds
# its targets_ / trackNumVec_ / timestamp_ and the UKF member functions to the instance already loaded by the test process.
REF      ?= /root/reference
OT       := $(REF)/object_tracking
OUT      := _ref
CXX      ?= g++
CXXFLAGS := -std=c++14 -O2 -w -fPIC
INC      := -I shim -I $(OT)/include -I $(OUT)/eigen_inc

.PHONY: all
all:
	@if [ -d "$(OT)" ]; then $(MAKE) --no-print-directory -f predict.mk $(OUT)/libref_predict_intended.so $(OUT)/libref_predict_tunable.so; \
	 else echo "oracle: $(REF) not present -- keeping prebuilt $(OUT)/libref_predict_*.so"; fi

$(OUT)/libref_predict_%.so: ref_predict.cpp $(OUT)/libref_%.so
	$(CXX) $(CXXFLAGS) $(INC) -shared -o $@ ref_predict.cpp -L $(OUT) -lref_$* -Wl,-rpath,'$$ORIGIN'
