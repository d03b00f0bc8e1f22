// mww_detector_records.h -- the packed detector record of mww_export_detector_rows / mww_import_detector_rows and the
// per-word bodies of the two kernels that fill and read it (mww_detector_records.cu).  One record holds one stream's rows
// of every used model of a detector (the plain detector: one WAKE model whose rows are its row indices):
//
//     uint64  member_mask                      bit k: the stream is a member of model k and slot k holds its state
//     for each model k whose role is not OFF:  float32 hist[window_k - 1]   oldest first (no bytes when window_k = 1)
//                                              int64 seen; int32 flag; int32 0   flag = cooldown (WAKE) or active (VAD)
//
// every part padded to 16 bytes.  detector_record_layout() is the only place that knows the offsets.  A record is moved a
// 4-byte word at a time; detector_record_pack_word / _unpack_word say what word w of a record holds and where it lives in
// the detector's struct-of-arrays state, as DetectModel describes it (hist [window - 1][n_rows], seen [n_rows],
// flag [n_rows], the inverse map [n_streams]).  CUDA-free apart from MWW_HD, so that tests/emul_detector_records.cc runs
// the same functions on the CPU.
#pragma once

#include <stdint.h>

#include "mww_detector_models.h"

namespace mww {

constexpr int kDetRecMaxModels = 64;          // one 64-bit member mask
constexpr int kDetRecMaskWords = 4;           // the mask and its padding: 16 bytes

inline long long detector_record_pad16(long long bytes) { return (bytes + 15) / 16 * 16; }

// byte offsets of each used model's history and of its seen / flag words; -1 for an OFF model
struct DetRecLayout {
    long long record_bytes;
    long long hist_off[kDetRecMaxModels], tail_off[kDetRecMaxModels];
};

// the offsets of the records of a detector whose models are models[0, n_models) (role and rule.window read)
inline DetRecLayout detector_record_layout(const DetectModel *models, int n_models) {
    DetRecLayout L{};
    long long off = detector_record_pad16(sizeof(uint64_t));
    for (int k = 0; k < n_models; ++k) {
        L.hist_off[k] = L.tail_off[k] = -1;
        if (models[k].role == MWW_DETECT_OFF) continue;
        L.hist_off[k] = off;
        off += detector_record_pad16((long long)(models[k].rule.window - 1) * (long long)sizeof(float));
        L.tail_off[k] = off;
        off += detector_record_pad16(sizeof(long long) + 2 * sizeof(int32_t));
    }
    L.record_bytes = off;
    return L;
}

// one used model as the kernels see it: its slot in the record (in words) and its rows' state
struct DetRecModel {
    int bit = 0;                     // the model's index k: its bit of the member mask
    int hist_word = 0, tail_word = 0;
    int hist_len = 0;                // window - 1
    int n_rows = 0;
    int fresh_flag = 0;              // what a reset gives: cooldown_slices (WAKE) or 0 (VAD)
    const int32_t *inv = nullptr;    // [n_ids]: row of each id, -1 for a non-member; nullptr: row = id
    float *hist = nullptr;
    long long *seen = nullptr;
    int32_t *flag = nullptr;
};

// every used model of a detector in record order, and the record's size in words
struct DetRecJob {
    int n_models = 0, words = 0;
    DetRecModel m[kDetRecMaxModels];
};

// the job of a detector whose models are models[0, n_models): a WAKE model's reset flag is its cooldown_slices
inline DetRecJob detector_record_job(const DetectModel *models, int n_models) {
    const DetRecLayout L = detector_record_layout(models, n_models);
    DetRecJob J;
    J.words = (int)(L.record_bytes / 4);
    for (int k = 0; k < n_models; ++k) {
        const DetectModel &s = models[k];
        if (s.role == MWW_DETECT_OFF) continue;
        DetRecModel &m = J.m[J.n_models++];
        m.bit = k;
        m.hist_word = (int)(L.hist_off[k] / 4);
        m.tail_word = (int)(L.tail_off[k] / 4);
        m.hist_len = s.rule.window - 1;
        m.n_rows = s.n_rows;
        m.fresh_flag = s.role == MWW_DETECT_WAKE ? s.rule.cooldown_slices : 0;
        m.inv = s.inv; m.hist = s.hist; m.seen = s.seen; m.flag = s.flag;
    }
    return J;
}

// model m's row of id (in range), -1 for a non-member
MWW_HD int detector_record_row(const DetRecModel &m, int id) { return m.inv ? m.inv[id] : id; }

// the used model whose slot holds word w (w >= kDetRecMaskWords): slots are in order and contiguous
MWW_HD int detector_record_model(const DetRecJob &J, int w) {
    int i = 0;
    while (i + 1 < J.n_models && w >= J.m[i + 1].hist_word) ++i;
    return i;
}

// where word w of model m's slot lives for row `row`: the state word it holds (written as the value), or nullptr for padding
// and the zero word; *fresh = its value in a reset row
MWW_HD uint32_t *detector_record_state_word(const DetRecModel &m, int w, int row, uint32_t *fresh) {
    *fresh = 0;
    if (w < m.tail_word) {
        const int j = w - m.hist_word;
        return j < m.hist_len ? reinterpret_cast<uint32_t *>(m.hist + (long long)j * m.n_rows + row) : nullptr;
    }
    const int t = w - m.tail_word;
    if (t < 2) return reinterpret_cast<uint32_t *>(m.seen + row) + t;          // little-endian halves of seen
    if (t == 2) { *fresh = (uint32_t)m.fresh_flag; return reinterpret_cast<uint32_t *>(m.flag + row); }
    return nullptr;
}

// detector -> record word w of the stream or row `id`.  The mask: a bit per used model the id is a member of.  A slot of a
// model the id is not a member of, padding and the zero word are written as zero.
MWW_HD void detector_record_pack_word(const DetRecJob &J, int w, int id, uint32_t *rec) {
    uint32_t v = 0;
    if (w < kDetRecMaskWords) {
        if (w < 2)
            for (int i = 0; i < J.n_models; ++i)
                if ((J.m[i].bit >> 5) == w && detector_record_row(J.m[i], id) >= 0) v |= 1u << (J.m[i].bit & 31);
    } else {
        const DetRecModel &m = J.m[detector_record_model(J, w)];
        const int row = detector_record_row(m, id);
        uint32_t fresh;
        if (row >= 0)
            if (const uint32_t *s = detector_record_state_word(m, w, row, &fresh)) v = *s;
    }
    rec[w] = v;
}

// record -> detector, word w.  Per used model: a non-member of the destination ignores the slot; a member whose mask bit is
// set takes the slot's word; a member whose bit is clear gets the reset value.  Padding and the mask are never written.
MWW_HD void detector_record_unpack_word(const DetRecJob &J, int w, int id, const uint32_t *rec) {
    if (w < kDetRecMaskWords) return;
    const DetRecModel &m = J.m[detector_record_model(J, w)];
    const int row = detector_record_row(m, id);
    if (row < 0) return;
    uint32_t fresh;
    uint32_t *s = detector_record_state_word(m, w, row, &fresh);
    if (!s) return;
    const bool has = (rec[m.bit >> 5] >> (m.bit & 31)) & 1u;
    *s = has ? rec[w] : fresh;
}

// The first field in which the layout the records were exported with differs from the importing detector's own, nullptr
// when the records fit.  *index = the model concerned for a per-model field, else -1.  A VAD's cooldown is not compared.
inline const char *detector_layout_mismatch(const mww_detector_layout &src, const mww_detector_layout &dst, int *index) {
    *index = -1;
    if (src.multi != dst.multi) return "multi";
    if (src.n_models != dst.n_models) return "n_models";
    for (int k = 0; k < dst.n_models && k < kDetRecMaxModels; ++k) {
        *index = k;
        if (src.role[k] != dst.role[k]) return "role";
        if (dst.role[k] != MWW_DETECT_OFF && src.window[k] != dst.window[k]) return "window";
        if (dst.role[k] == MWW_DETECT_WAKE && src.cooldown_slices[k] != dst.cooldown_slices[k]) return "cooldown_slices";
    }
    *index = -1;
    if (src.record_bytes != dst.record_bytes) return "record_bytes";
    return nullptr;
}

}  // namespace mww
