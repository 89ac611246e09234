# TEST INFRASTRUCTURE ONLY -- builds oracle/_ref/libref_tunable.so: libref_intended.so (see Makefile) with the tracker's constants
# read from globals a test can set (oracle/ref_tunable.py), so that lmot_tracker_params can be checked against the reference itself.
#
#   make -f tunable.mk   (after `make ref`, whose box_fitting_intended.cpp and Eigen link it reuses)
#
# Build-time copies of imm_ukf_jpda.cpp and ukf.cpp, patched by sed; every pattern is checked to apply exactly as often as expected
# (count of the patched text in the copy).  Nothing of the reference is committed: the copies live in _ref/ only.
#   imm_ukf_jpda.cpp  the six `const` file-scope constants (:26-45) become plain exported globals; the static-object thresholds
#                     (:1064, :1067) and the second-init speed (:902) read globals of tunable_params.cpp
#   ukf.cpp           the constructor's process / lidar noise (:68-94), transition rows (:144-154), mode probabilities (:180-182)
#                     and the P_merge_ initialiser (:275-279) read globals of tunable_params.cpp
REF      ?= /root/reference
OT       := $(REF)/object_tracking
OUT      := _ref
CXX      ?= g++
CXXFLAGS := -std=c++14 -O2 -w -fPIC
INC      := -I shim -I $(OT)/include -I $(OUT)/eigen_inc
UNPATCHED := $(OT)/src/groundremove/ground_removal.cpp $(OT)/src/groundremove/gaus_blur.cpp $(OT)/src/cluster/component_clustering.cpp

.PHONY: all
all:
	@if [ -d "$(OT)" ]; then $(MAKE) --no-print-directory -f tunable.mk $(OUT)/libref_tunable.so; \
	 else echo "oracle: $(REF) not present -- keeping prebuilt $(OUT)/libref_tunable.so"; fi

# count(file, fixed string, n): the patched text occurs exactly n times
count = @test `grep -cF '$(2)' $(1)` -eq $(3) || (echo "$(1): '$(2)' expected $(3) times"; rm -f $(1); exit 1)

$(OUT)/imm_ukf_jpda_tunable.cpp: $(OT)/tracking/imm_ukf_jpda.cpp
	mkdir -p $(OUT)
	sed -e 's/^const \(double\|int\) \(gammaG_\|pG_\|pD_\|distanceThres_\|lifeTimeThres_\|bbYawChangeThres_\) /\1 \2 /' \
	    -e 's/targets_\[i\]\.lifetime_ > 8 )/targets_[i].lifetime_ > lmot_tp_static_lifetime )/' \
	    -e 's/^\(\s*\)distThres = 3\.0;/\1distThres = lmot_tp_static_dist;/' \
	    -e 's/double targetV   = 2;/double targetV   = lmot_tp_second_init_v;/' \
	    -e '1i extern "C" { extern int lmot_tp_static_lifetime; extern double lmot_tp_static_dist, lmot_tp_second_init_v; }' \
	    $< > $@
	$(call count,$@,extern "C" { extern int lmot_tp_static_lifetime;,1)
	@test `grep -cE '^(double gammaG_|double pG_|double pD_|double distanceThres_|int lifeTimeThres_|double bbYawChangeThres_) ' $@` -eq 6 || \
	  (echo "$@: the six constants did not all lose their const"; rm -f $@; exit 1)
	$(call count,$@,lifetime_ > lmot_tp_static_lifetime,1)
	$(call count,$@,distThres = lmot_tp_static_dist;,1)
	$(call count,$@,targetV   = lmot_tp_second_init_v;,1)
	@test `diff $< $@ | grep -c "^>"` -eq 10 || (echo "$@: unexpected changes"; rm -f $@; exit 1)

$(OUT)/ukf_tunable.cpp: $(OT)/tracking/ukf.cpp
	mkdir -p $(OUT)
	sed -e 's/^\(\s*\)std_a_cv_ *= 2;/\1std_a_cv_ = lmot_tp_std_a[0];/' \
	    -e 's/^\(\s*\)std_a_ctrv_ *= 2;/\1std_a_ctrv_ = lmot_tp_std_a[1];/' \
	    -e 's/^\(\s*\)std_a_rm_ *= 3;/\1std_a_rm_ = lmot_tp_std_a[2];/' \
	    -e 's/^\(\s*\)std_cv_yawdd_ *= 2;/\1std_cv_yawdd_ = lmot_tp_std_yawdd[0];/' \
	    -e 's/^\(\s*\)std_ctrv_yawdd_ *= 2;/\1std_ctrv_yawdd_ = lmot_tp_std_yawdd[1];/' \
	    -e 's/^\(\s*\)std_rm_yawdd_ *= 3;/\1std_rm_yawdd_ = lmot_tp_std_yawdd[2];/' \
	    -e 's/^\(\s*\)std_laspx_ = 0\.15;/\1std_laspx_ = lmot_tp_std_las[0];/' \
	    -e 's/^\(\s*\)std_laspy_ = 0\.15;/\1std_laspy_ = lmot_tp_std_las[1];/' \
	    -e 's/^\(\s*\)p\([123]\)_\.push_back([0-9.]*);/\1p\2_.push_back(lmot_tp_trans[\2 - 1][p\2_.size()]);/' \
	    -e 's/^\(\s*\)modeProbCV_ = 0\.33;/\1modeProbCV_ = lmot_tp_mode_prob0[0];/' \
	    -e 's/^\(\s*\)modeProbCTRV_ = 0\.33;/\1modeProbCTRV_ = lmot_tp_mode_prob0[1];/' \
	    -e 's/^\(\s*\)modeProbRM_ = 0\.33;/\1modeProbRM_ = lmot_tp_mode_prob0[2];/' \
	    -e '/^    P_merge_ <<   0\.5,/,/;/c\' \
	    -e '    P_merge_ << lmot_tp_p0_diag[0], 0, 0, 0, 0,  0, lmot_tp_p0_diag[1], 0, 0, 0,  0, 0, lmot_tp_p0_diag[2], 0, 0,  0, 0, 0, lmot_tp_p0_diag[3], 0,  0, 0, 0, 0, lmot_tp_p0_diag[4];' \
	    -e '1i extern "C" { extern double lmot_tp_std_a[3], lmot_tp_std_yawdd[3], lmot_tp_std_las[2], lmot_tp_trans[3][3], lmot_tp_mode_prob0[3], lmot_tp_p0_diag[5]; }' \
	    $< > $@
	$(call count,$@,extern "C" { extern double lmot_tp_std_a[3],1)
	$(call count,$@,= lmot_tp_std_a[,3)
	$(call count,$@,= lmot_tp_std_yawdd[,3)
	$(call count,$@,= lmot_tp_std_las[,2)
	$(call count,$@,][p,9)
	$(call count,$@,= lmot_tp_mode_prob0[,3)
	$(call count,$@,P_merge_ << lmot_tp_p0_diag[0],1)
	@test `diff $< $@ | grep -c "^>"` -eq 24 || (echo "$@: unexpected changes"; rm -f $@; exit 1)
	@test `diff $< $@ | grep -c "^<"` -eq 27 || (echo "$@: unexpected removals"; rm -f $@; exit 1)

$(OUT)/box_fitting_intended.cpp $(OUT)/eigen_inc/Eigen:
	$(MAKE) --no-print-directory -f Makefile $@

$(OUT)/libref_tunable.so: ref_harness.cpp mar_contract.cpp tunable_params.cpp $(OUT)/imm_ukf_jpda_tunable.cpp $(OUT)/ukf_tunable.cpp \
                          $(OUT)/box_fitting_intended.cpp $(OUT)/eigen_inc/Eigen
	$(CXX) $(CXXFLAGS) -DLMOT_REF_INTENDED $(INC) -shared -o $@ $(UNPATCHED) $(OUT)/ukf_tunable.cpp $(OUT)/imm_ukf_jpda_tunable.cpp \
	  $(OUT)/box_fitting_intended.cpp ref_harness.cpp mar_contract.cpp tunable_params.cpp
