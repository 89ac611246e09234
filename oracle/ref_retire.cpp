// TEST INFRASTRUCTURE ONLY -- track retirement on the reference's own track table (lmot_set_track_retirement's oracle).
//
// Built by oracle/retire.mk into oracle/_ref/libref_retire_<mode>.so, one per reference library (intended, tunable), each linked
// against its libref_<mode>.so: loaded after that library, it resolves targets_ / trackNumVec_ to the SAME instance the harness
// (ref_harness.cpp) steps, so that a test can interleave ref_tracker_step and ref_tracker_retire on one table.
// No algorithm of the reference is restated here: the function only erases entries of its two containers.
#include <vector>
#include "ukf.h"

// the track table: externally linked globals of imm_ukf_jpda.cpp:57-58
extern std::vector<UKF> targets_;
extern std::vector<int> trackNumVec_;

extern "C" {

// stably erase every i with trackNumVec_[i] == 0 from targets_ and trackNumVec_.  Nothing else changes: the ego fold (egoPoints_,
// egoDeltaHis_), init_ and timestamp_ stay as immUkfJpdaf left them (unlike ref_tracker_load, which restarts the fold).
void ref_tracker_retire() {
  size_t w = 0;
  for (size_t i = 0; i < targets_.size(); ++i) {
    if (trackNumVec_[i] == 0) continue;
    if (w != i) { targets_[w] = targets_[i]; trackNumVec_[w] = trackNumVec_[i]; }
    ++w;
  }
  targets_.erase(targets_.begin() + w, targets_.end());
  trackNumVec_.erase(trackNumVec_.begin() + w, trackNumVec_.end());
}

}  // extern "C"
