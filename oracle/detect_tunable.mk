# TEST INFRASTRUCTURE ONLY -- builds oracle/_ref/libref_detect_tunable.so: libref_intended.so (see Makefile) with the two detection
# literals read from globals a test can set, so that lmot_detect_params.ground_tolerance and min_cluster_points can be checked against
# the reference itself (every other detection value is a mutable global of the reference already).
#
#   make -f detect_tunable.mk   (after `make ref`, whose box_fitting_intended.cpp and Eigen link it reuses)
#
# Build-time copies, patched by sed; every pattern is checked to apply exactly as often as expected.  Nothing of the reference is
# committed: the copies live in _ref/ only.
#   ground_removal.cpp        `z < (hGround + 0.25)` (:239) reads lmot_dp_ground_tolerance (double, as the literal)
#   box_fitting_intended.cpp  `numPoints < 30` (:100) reads lmot_dp_min_cluster_points
# The globals and their defaults are in detect_tunable_params.cpp.
REF      ?= /root/reference
OT       := $(REF)/object_tracking
OUT      := _ref
CXX      ?= g++
CXXFLAGS := -std=c++14 -O2 -w -fPIC
INC      := -I shim -I $(OT)/include -I $(OUT)/eigen_inc
UNPATCHED := $(OT)/src/groundremove/gaus_blur.cpp $(OT)/src/cluster/component_clustering.cpp $(OT)/tracking/ukf.cpp \
             $(OT)/tracking/imm_ukf_jpda.cpp

.PHONY: all
all:
	@if [ -d "$(OT)" ]; then $(MAKE) --no-print-directory -f detect_tunable.mk $(OUT)/libref_detect_tunable.so; \
	 else echo "oracle: $(REF) not present -- keeping prebuilt $(OUT)/libref_detect_tunable.so"; fi

# count(file, fixed string, n): the patched text occurs exactly n times
count = @test `grep -cF '$(2)' $(1)` -eq $(3) || (echo "$(1): '$(2)' expected $(3) times"; rm -f $(1); exit 1)

$(OUT)/ground_removal_detect_tunable.cpp: $(OT)/src/groundremove/ground_removal.cpp
	mkdir -p $(OUT)
	sed -e 's/if (z < (hGround + 0\.25)) {/if (z < (hGround + lmot_dp_ground_tolerance)) {/' \
	    -e '1i extern "C" { extern double lmot_dp_ground_tolerance; }' \
	    $< > $@
	$(call count,$@,extern "C" { extern double lmot_dp_ground_tolerance; },1)
	$(call count,$@,(hGround + lmot_dp_ground_tolerance),1)
	$(call count,$@,hGround + 0.25,0)
	@test `diff $< $@ | grep -c "^>"` -eq 2 || (echo "$@: unexpected changes"; rm -f $@; exit 1)

$(OUT)/box_fitting_detect_tunable.cpp: $(OUT)/box_fitting_intended.cpp
	sed -e 's/if(numPoints < 30) return isPromising;/if(numPoints < lmot_dp_min_cluster_points) return isPromising;/' \
	    -e '1i extern "C" { extern int lmot_dp_min_cluster_points; }' \
	    $< > $@
	$(call count,$@,extern "C" { extern int lmot_dp_min_cluster_points; },1)
	$(call count,$@,numPoints < lmot_dp_min_cluster_points,1)
	$(call count,$@,numPoints < 30,0)
	@test `diff $< $@ | grep -c "^>"` -eq 2 || (echo "$@: unexpected changes"; rm -f $@; exit 1)

$(OUT)/box_fitting_intended.cpp $(OUT)/eigen_inc/Eigen:
	$(MAKE) --no-print-directory -f Makefile $@

$(OUT)/libref_detect_tunable.so: ref_harness.cpp mar_contract.cpp detect_tunable_params.cpp $(OUT)/ground_removal_detect_tunable.cpp \
                                 $(OUT)/box_fitting_detect_tunable.cpp $(OUT)/eigen_inc/Eigen
	$(CXX) $(CXXFLAGS) -DLMOT_REF_INTENDED $(INC) -I $(OT)/src/groundremove -shared -o $@ $(UNPATCHED) \
	  $(OUT)/ground_removal_detect_tunable.cpp $(OUT)/box_fitting_detect_tunable.cpp ref_harness.cpp mar_contract.cpp detect_tunable_params.cpp
