// enc_refs.h — per-stream reference picture management of the encoder: which picture a P picture predicts from, which slot
// of the stream's picture store it reconstructs into, the slice header's list modification and marking syntax, and the
// long-term reference (LTR) state that loss-recovery feedback drives.  Host only and free of CUDA, so that the decisions can be
// checked without a device (tests/test_enc_refs_cpu.py).
//
// Behavioural model: the camera path of the reference's codec/encoder/core/src/ref_list_mgr_svc.cpp with one spatial and one
// temporal layer (GOP size 1): WelsMarkPic (:494), WelsBuildRefList (:594), WelsUpdateRefSyntax (:662-726), WelsUpdateRefList
// (:357) with LTRMarkProcess (:251), DeleteInvalidLTR (:160) and HandleLTRMarkFeedback (:195), and the feedback filters
// FilterLTRRecoveryRequest / FilterLTRMarkingFeedback (:517, :563).  The reference's list bookkeeping is kept literally,
// including its index walks that skip the entry behind a deleted one, because what it deletes decides later pictures.
// The source pictures the LOW_COMPLEXITY VAA statistics compare against follow CWelsPreProcess (wels_preprocess.cpp:263-335).
#pragma once
#include <stdint.h>

namespace b2h264 {

// values of the reference's public API (codec_app_def.h)
enum { kLtrRecoveryRequest = 1, kLtrMarkingSuccess = 4, kLtrMarkingFailed = 5 };
enum { kLongTermRefNum = 2,                  // LONG_TERM_REF_NUM (camera)
       kMaxNumRefFramesCamera = 10 };        // MAX_REFERENCE_PICTURE_COUNT_NUM_CAMERA

// The reference configuration resolved as the reference resolves it for one temporal layer (au_set.cpp:88-133,
// param_svc.h:376-385): `requested` is what the caller asked for (AUTO_REF_PIC_COUNT = -1, or 1..10).
struct RefConfig {
  bool ltr = false;
  int ltr_mark_period = 30;
  int sps_num_ref_frames = 1;                // max_num_ref_frames of the SPS (iMaxNumRefFrame)
  int num_ref_frames = 1;                    // iNumRefFrame as the encoder reports it
  int ltr_ref_num = 0;                       // iLTRRefNum as the encoder reports it
  // pictures of the device store per stream: the one reconstructed into plus the ones kept.  Without LTR the reference keeps
  // only the newest short-term picture whatever max_num_ref_frames says; with LTR it keeps at most one short-term and two
  // long-term pictures.
  int slots() const { return ltr ? 2 + kLongTermRefNum : 2; }
  // source pictures per stream for the VAA statistics: current, previous and one per long-term index
  int src_slots() const { return ltr ? 2 + kLongTermRefNum : 2; }
  static bool resolve(int requested, bool ltr, int ltr_mark_period, int intra_period, RefConfig* out) {
    if (requested != -1 && (requested < 1 || requested > kMaxNumRefFramesCamera)) return false;
    RefConfig c;
    c.ltr = ltr;
    c.ltr_mark_period = ltr_mark_period == 0 ? 30 : ltr_mark_period;   // iLtrMarkPeriod 0: the default (welsEncoderExt.cpp:321-323)
    c.ltr_ref_num = ltr ? kLongTermRefNum : 0;
    int needed = intra_period != 1 ? 1 + c.ltr_ref_num : 0;
    needed = needed < 1 ? 1 : (needed > kMaxNumRefFramesCamera ? kMaxNumRefFramesCamera : needed);
    int n = requested == -1 || requested < needed ? needed : requested;
    c.sps_num_ref_frames = n;
    c.num_ref_frames = needed;
    *out = c;
    return true;
  }
};

// What one picture needs from the reference state: where its pictures are and what its slice header says.
struct RefDecision {
  bool idr = false;
  bool not_coded = false;                    // no picture to predict from: the picture is dropped and the next one is an IDR
  int frame_num = 0;
  int idr_pic_id = 0;
  int rec_slot = 0;                          // store slot reconstructed into
  int ref_slot = -1;                         // store slot of the reference picture (P)
  bool ref_is_p = false;                     // the reference picture was coded as a P picture
  int mod_idc = 0, mod_val = 0;              // ref_pic_list_modification: idc 0 + abs_diff_pic_num_minus1, or idc 2 + long_term_pic_num
  bool long_term_reference_flag = false;     // IDR
  int n_mmco = 0;                            // P: adaptive_ref_pic_marking_mode_flag = n_mmco > 0
  int mmco[3][3] = {};                       // memory_management_control_operation, first value, second value (op 3)
  int cur_src = 0, vaa_src = 0;              // source slots: this picture's, and the one its VAA statistics compare against
};

class StreamRefs {
 public:
  RefConfig cfg;

  void reset() {
    const RefConfig keep = cfg;
    *this = StreamRefs();
    cfg = keep;
    for (int i = 0; i < 2 + kLongTermRefNum; i++) src_[i] = i;
    src_[0] = 1; src_[1] = 0;                 // the first picture's source lands in slot 0
  }
  StreamRefs() { for (int i = 0; i < 2 + kLongTermRefNum; i++) src_[i] = i; src_[0] = 1; src_[1] = 0; }

  // the state asks for the next picture to be an IDR (bEncCurFrmAsIdrFlag set by feedback or by losing every long-term picture)
  bool idr_wanted() const { return want_idr_; }
  int idr_pic_id() const { return idr_pic_id_; }
  int last_rec_slot() const { return last_rec_; }

  // decisions for the next picture, and the state after it (the state does not depend on what the picture's content is)
  RefDecision code_picture(bool idr) {
    RefDecision d;
    want_idr_ = false;
    const int fn = idr ? 0 : frame_num_;
    if (idr) idr_pic_id_ = idr_pic_id_ < 65535 ? idr_pic_id_ + 1 : 0;
    d.idr = idr; d.frame_num = fn; d.idr_pic_id = idr_pic_id_;
    d.cur_src = src_[1];
    d.vaa_src = t0_lost_ ? src_[2 + valid_lt_idx_] : src_[0];
    mark_pic(d, fn);
    // WelsBuildRefList
    const Pic* ref = nullptr;
    if (!idr) {
      if (cfg.ltr && t0_lost_) {
        for (int i = 0; i < n_lt_; i++)
          if (lt_[i].confirmed) { ref = &lt_[i]; last_recover_fn_ = fn; break; }
      } else if (n_st_ > 0) {
        ref = &st_[0];
      }
    } else {
      n_st_ = n_lt_ = 0;
      reset_ltr();
    }
    if (!idr && !ref) {
      // a recovery request with no confirmed long-term picture left: the reference's WelsBuildRefList fails, the picture is not
      // coded (EncodeFrame returns cmUnknownReason), the source pictures still rotate and the next picture is an IDR
      // (encoder_ext.cpp:3630-3636, 4099-4106: UpdateSpatialPictures, ForceCodingIDR)
      d.not_coded = true;
      update_sources(false);
      frame_num_ = 0;
      want_idr_ = true;
      return d;
    }
    // WelsUpdateRefSyntax
    if (ref) {
      d.ref_slot = ref->slot;
      d.ref_is_p = ref->is_p;
      if (!ref->is_long || !cfg.ltr) {
        int diff = fn - ref->frame_num - 1;
        if (diff < 0) diff += kMaxFrameNum;
        d.mod_idc = 0; d.mod_val = diff;
      } else {
        d.mod_idc = 2; d.mod_val = ref->lt_pic_num;
      }
    }
    if (idr) { d.long_term_reference_flag = cfg.ltr; d.n_mmco = 0; }
    // the slot to reconstruct into: the first one no list holds (PrefetchNextBuffer)
    for (int s = 0; s < cfg.slots(); s++) {
      bool used = false;
      for (int i = 0; i < n_st_; i++) used |= st_[i].slot == s;
      for (int i = 0; i < n_lt_; i++) used |= lt_[i].slot == s;
      if (!used) { d.rec_slot = s; break; }
    }
    last_rec_ = d.rec_slot;
    update_ref_list(d, fn);
    update_sources(idr);
    frame_num_ = fn < kMaxFrameNum - 1 ? fn + 1 : 0;
    return d;
  }

  // ENCODER_LTR_RECOVERY_REQUEST (FilterLTRRecoveryRequest)
  void recovery_request(int type, int idr_pic_id, int cur_fn, int last_correct_fn) {
    if (!cfg.ltr) { want_idr_ = true; return; }
    if (type != kLtrRecoveryRequest || idr_pic_id != idr_pic_id_) return;
    if (last_correct_fn == -1) { want_idr_ = true; return; }
    if (cur_fn == -1) { t0_lost_ = true; return; }
    if ((cmp(last_recover_fn_, last_correct_fn) & (kEqual | kSmaller)) ||
        ((cmp(last_recover_fn_, cur_fn) & (kEqual | kSmaller)) && cmp(last_recover_fn_, last_correct_fn) == kBigger)) {
      t0_lost_ = true;
      last_cor_fn_dec_ = last_correct_fn;
      cur_fn_in_dec_ = cur_fn;
    }
  }
  // ENCODER_LTR_MARKING_FEEDBACK (FilterLTRMarkingFeedback)
  void marking_feedback(int type, int idr_pic_id, int ltr_fn) {
    if (!cfg.ltr) return;
    if (idr_pic_id == idr_pic_id_ && (type == kLtrMarkingSuccess || type == kLtrMarkingFailed)) {
      mark_state_ = type;
      mark_fb_fn_ = ltr_fn;
    }
  }
  // ENCODER_LTR_MARKING_PERIOD
  void set_mark_period(int period) { cfg.ltr_mark_period = period; }

 private:
  enum { kEqual = 1, kBigger = 2, kSmaller = 4 };
  enum { kDirect = 0, kDelay = 1 };
  static constexpr int kMaxFrameNum = 1 << 15;   // log2_max_frame_num 15 (h264_bitstream.cpp: write_sps)
  struct Pic { int slot, frame_num, mark_frame_num, lt_pic_num; bool is_long, confirmed, is_p; };

  // CompareFrameNum (ref_list_mgr_svc.cpp:118)
  static int cmp(int a, int b) {
    if (a > kMaxFrameNum || b > kMaxFrameNum) return -2;
    auto ad = [](int64_t x, int64_t y) { return x > y ? x - y : y - x; };
    const int64_t d = ad(a, b);
    if (d == 0) return kEqual;
    const int64_t na = ad((int64_t)a + kMaxFrameNum, b);
    if (na == 0) return kEqual;
    if (d > na) return kBigger;
    const int64_t nb = ad((int64_t)b + kMaxFrameNum, a);
    if (nb == 0) return kEqual;
    if (d > nb) return kSmaller;
    return a > b ? kBigger : kSmaller;
  }
  static void erase(Pic* l, int* n, int i) { for (int k = i; k < *n - 1; k++) l[k] = l[k + 1]; (*n)--; }

  void reset_ltr() {                          // ResetLtrState
    t0_lost_ = false; last_recover_fn_ = 0; last_cor_fn_dec_ = -1; cur_fn_in_dec_ = -1;
    mark_mode_ = kDirect; success_num_ = 0; marking_ = false; mark_enable_ = false; cur_ltr_idx_ = 0; mark_interval_ = 0;
    mark_state_ = 0; mark_fb_fn_ = -1;
  }

  // WelsMarkPic + WelsMarkMMCORefInfo (GOP size 1: the short-term picture to turn long is always one picture back)
  void mark_pic(RefDecision& d, int fn) {
    if (cfg.ltr && mark_enable_) {
      bool used = false;                      // CheckCurMarkFrameNumUsed
      for (int i = 0; i < n_lt_; i++)
        if ((fn == lt_[i].frame_num && mark_mode_ == kDirect) || (cmp(fn + 1, lt_[i].frame_num) == kEqual && mark_mode_ == kDelay)) used = true;
      if (!t0_lost_ && mark_interval_ > (uint32_t)cfg.ltr_mark_period && !used) {
        marking_ = true; mark_enable_ = false; mark_interval_ = 0;
      } else {
        marking_ = false;
      }
    }
    d.n_mmco = 0;
    if (cfg.ltr && marking_) {
      if (mark_mode_ == kDirect) {
        d.mmco[0][0] = 4; d.mmco[0][1] = kLongTermRefNum - 1 + 1;       // max_long_term_frame_idx_plus1
        d.mmco[1][0] = 1; d.mmco[1][1] = 1 - 1;                         // difference_of_pic_nums_minus1
        d.mmco[2][0] = 6; d.mmco[2][1] = cur_ltr_idx_;                  // long_term_frame_idx
        d.n_mmco = 3;
      } else {
        d.mmco[0][0] = 3; d.mmco[0][1] = 1 - 1; d.mmco[0][2] = cur_ltr_idx_;
        d.n_mmco = 1;
      }
    }
  }

  // WelsUpdateRefList: the new picture goes to the front of the short-term list, then marking and feedback
  void update_ref_list(const RefDecision& d, int fn) {
    for (int i = n_st_; i > 0; i--) st_[i] = st_[i - 1];
    st_[0] = Pic{d.rec_slot, fn, 0, 0, false, false, !d.idr};
    n_st_++;
    if (!d.idr) {
      if (cfg.ltr) {
        ltr_mark_process(false, fn);
        delete_invalid_ltr();
        handle_mark_feedback();
        t0_lost_ = false;
        marking_ = false;
        ++mark_interval_;
      }
      for (int i = n_st_ - 1; i > 0; i--) erase(st_, &n_st_, i);
      if (n_st_ > 0 && st_[0].frame_num != fn) erase(st_, &n_st_, 0);
    } else if (cfg.ltr) {
      ltr_mark_process(true, fn);
      cur_ltr_idx_ = (cur_ltr_idx_ + 1) % kLongTermRefNum;
      success_num_ = 1;
      mark_enable_ = true;
      mark_interval_ = 0;
      valid_lt_idx_ = 0;
      mark_lt_idx_ = 0;
    }
  }

  void ltr_mark_process(bool islice, int fn) {  // LTRMarkProcess
    int i = 0;
    if (islice) {
      st_[0].confirmed = true;
    } else if (marking_) {
      mark_lt_idx_ = cur_ltr_idx_;
      if (mark_mode_ == kDelay)
        for (i = 0; i < n_st_; i++)
          if (cmp(fn, st_[i].frame_num + 1) == kEqual) break;
    }
    if (islice || marking_) {
      st_[i].is_long = true;
      st_[i].lt_pic_num = cur_ltr_idx_;
      st_[i].mark_frame_num = fn;
    }
    bool move = false;
    if (mark_mode_ == kDirect && !islice && !marking_)
      for (int j = 0; j < n_st_; j++)
        if (st_[j].is_long) { i = j; move = true; break; }
    if ((mark_mode_ == kDelay && marking_) || (mark_mode_ == kDirect && move)) {
      ref_of_cur_is_ltr_ = true;
      for (int k = n_lt_; k > 0; k--) lt_[k] = lt_[k - 1];
      lt_[0] = st_[i];
      n_lt_++;
      if (n_lt_ > kLongTermRefNum) erase(lt_, &n_lt_, n_lt_ - 1);
      erase(st_, &n_st_, i);
    }
  }

  void delete_invalid_ltr() {                 // DeleteInvalidLTR
    for (int i = 0; i < kLongTermRefNum; i++) {
      if (i >= n_lt_) continue;
      const Pic& p = lt_[i];
      const bool bad_fn = cmp(p.frame_num, last_cor_fn_dec_) == kBigger && (cmp(p.frame_num, cur_fn_in_dec_) & (kEqual | kSmaller));
      const bool bad_mark = cmp(p.mark_frame_num, last_cor_fn_dec_) == kBigger &&
                            (cmp(p.mark_frame_num, cur_fn_in_dec_) & (kEqual | kSmaller)) && mark_mode_ == kDelay;
      if (bad_fn || bad_mark) {
        erase(lt_, &n_lt_, i);
        mark_enable_ = true;
        if (n_lt_ == 0) want_idr_ = true;
      }
    }
  }

  void handle_mark_feedback() {               // HandleLTRMarkFeedback
    if (mark_state_ == kLtrMarkingSuccess) {
      for (int i = 0; i < n_lt_; i++) {
        if (lt_[i].frame_num == mark_fb_fn_ && !lt_[i].confirmed) {
          lt_[i].confirmed = true;
          valid_lt_idx_ = lt_[i].lt_pic_num;
          cur_fn_in_dec_ = last_recover_fn_ = last_cor_fn_dec_ = mark_fb_fn_;
          for (int j = 0; j < n_lt_; j++)
            if (lt_[j].lt_pic_num != cur_ltr_idx_) erase(lt_, &n_lt_, j);
          success_num_++;
          cur_ltr_idx_ = (cur_ltr_idx_ + 1) % kLongTermRefNum;
          mark_mode_ = success_num_ >= kLongTermRefNum ? kDelay : kDirect;
          mark_enable_ = true;
          break;
        }
      }
      mark_state_ = 0;
    } else if (mark_state_ == kLtrMarkingFailed) {
      for (int i = 0; i < n_lt_; i++)
        if (lt_[i].frame_num == mark_fb_fn_) { erase(lt_, &n_lt_, i); break; }
      mark_state_ = 0;
      mark_enable_ = true;
      if (success_num_ == 0) want_idr_ = true;
    }
  }

  // CWelsPreProcess::UpdateSpatialPictures after the picture, then the flag WelsEncoderEncodeExt sets for the next one
  // (encoder_ext.cpp:4084: after WelsUpdateRefList has cleared bLTRMarkingFlag of a P picture only an IDR sets it)
  void update_sources(bool idr) {
    if (ref_of_cur_is_ltr_) {
      const int k = 2 + mark_lt_idx_, t = src_[k];
      src_[k] = src_[0]; src_[0] = t;
      ref_of_cur_is_ltr_ = false;
    }
    const int t = src_[1]; src_[1] = src_[0]; src_[0] = t;
    if (cfg.ltr && idr) ref_of_cur_is_ltr_ = true;
  }

  Pic st_[3 + kLongTermRefNum] = {}, lt_[kLongTermRefNum + 1] = {};
  int n_st_ = 0, n_lt_ = 0;
  int frame_num_ = 0, idr_pic_id_ = 0, last_rec_ = 1;
  bool want_idr_ = false;
  // SLTRState
  bool t0_lost_ = false, marking_ = false, mark_enable_ = false;
  int last_recover_fn_ = 0, last_cor_fn_dec_ = -1, cur_fn_in_dec_ = -1;
  int mark_mode_ = kDirect, success_num_ = 0, cur_ltr_idx_ = 0;
  uint32_t mark_interval_ = 0;
  int mark_state_ = 0, mark_fb_fn_ = -1;
  int valid_lt_idx_ = 0, mark_lt_idx_ = 0;    // SVAAFrameInfo::uiValidLongTermPicIdx / uiMarkLongTermPicIdx
  bool ref_of_cur_is_ltr_ = false;            // bRefOfCurTidIsLtr
  int src_[2 + kLongTermRefNum];              // m_pSpatialPic: [0] previous source, [1] current, [2 + i] long-term index i
};

}  // namespace b2h264
