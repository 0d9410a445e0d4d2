// tests/ref_kfdb.cpp — TEST INFRASTRUCTURE ONLY.
//
// A C entry point over the reference's own KeyFrameDatabase (src/KeyFrameDatabase.cc) and DBoW2 L1 scoring, as compiled into
// oracle/_ref/libref.so.  tests/test_kfdb_cpu.py compiles this file against the reference's headers and the stand-ins of oracle/refshim/
// with the flags of oracle/ref_build.sh, links it with libref.so, and holds tests/kfdb_model.py to it.
#include <chrono>
#include <cmath>
#include <cstdint>
#include <map>
#include <vector>
#include "refshim/minicv.hpp"

#define private public
#define protected public
#include "Frame.h"
#include "KeyFrame.h"
#include "Map.h"
#include "KeyFrameDatabase.h"
#include "ORBVocabulary.h"
#undef private
#undef protected

using namespace StructureSLAM;

namespace {

DBoW2::BowVector bow(const int32_t* off, const int32_t* word, const double* val, int r) {
    DBoW2::BowVector v;
    for (int i = off[r]; i < off[r + 1]; i++) v[word[i]] = val[i];
    return v;
}

// A Frame without features: what KeyFrameDatabase reads of frames and keyframes is mBowVec, mnId and the covisibility fields.
Frame* empty_frame(ORBVocabulary* voc) {
    Frame* F = new Frame();
    F->mpORBvocabulary = voc; F->mpORBextractorLeft = nullptr; F->mpORBextractorRight = nullptr; F->mpLineSegment = nullptr;
    F->mTimeStamp = 0; F->mbf = 0; F->mb = 0; F->mThDepth = 0; F->mpReferenceKF = nullptr; F->dealWithLine = false; F->blurNumber = 0;
    F->mnId = Frame::nNextId++;
    F->N = 0; F->NL = 0; F->mnScaleLevels = 1; F->mfScaleFactor = 1.f; F->mfLogScaleFactor = 0.f;
    F->mvScaleFactors.assign(1, 1.f); F->mvInvScaleFactors.assign(1, 1.f); F->mvLevelSigma2.assign(1, 1.f); F->mvInvLevelSigma2.assign(1, 1.f);
    F->mK = cv::Mat::eye(3, 3, CV_32F); F->mDistCoef = cv::Mat::zeros(4, 1, CV_32F);
    F->SetPose(cv::Mat::eye(4, 4, CV_32F));
    return F;
}

}  // namespace

extern "C" {

/* TemplatedVocabulary::score (L1Scoring::score) of row pairs (pair[2 i], pair[2 i + 1]) of the BowVectors (word, val)[off[r] .. off[r + 1]). */
void ref_bow_score(void* voc, const int32_t* off, const int32_t* word, const double* val, int npairs, const int32_t* pair, double* out) {
    ORBVocabulary* V = static_cast<ORBVocabulary*>(voc);
    for (int i = 0; i < npairs; i++) out[i] = V->score(bow(off, word, val, pair[2 * i]), bow(off, word, val, pair[2 * i + 1]));
}

/* nrows keyframes: BowVector of row r = (word, val)[off[r] .. off[r + 1]), GetBestCovisibilityKeyFrames = covis[r][0 .. ncovis[r]),
   mConnectedKeyFrameWeights = the rows conn[conn_off[r] .. conn_off[r + 1]), mLoopScore = 0 and mRelocScore = relocscore[r].  The rows
   add[0 .. nadd) are added to a KeyFrameDatabase on the vocabulary voc (ref.Vocabulary's handle) in that order, then erase[0 .. nerase)
   are erased.  Then nq queries run in sequence: loop: DetectLoopCandidates(keyframe query[q], minscore[q]); reloc: a Frame with row
   query[q]'s BowVector and a fresh id, DetectRelocalizationCandidates(F).  Out per query q: cand[q][0 .. ncand[q]) as rows, and per row
   r: words[q][r] = mnLoopWords / mnRelocWords when the keyframe carries the query's id (0 otherwise), score[q][r] = mLoopScore /
   mRelocScore after the query; *seconds (may be NULL) = the wall time of the nq queries. */
void ref_kfdb_query(void* voc, int nrows, const int32_t* off, const int32_t* word, const double* val, const int32_t* covis, const int32_t* ncovis,
                    const int32_t* conn_off, const int32_t* conn, const float* relocscore, int nadd, const int32_t* add, int nerase,
                    const int32_t* erase, int loop, int nq, const int32_t* query, const float* minscore,
                    int32_t* cand, int32_t* ncand, int32_t* words, float* score, double* seconds) {
    ORBVocabulary* V = static_cast<ORBVocabulary*>(voc);
    Map map;
    KeyFrameDatabase db(*V);
    std::vector<Frame*> frames;
    std::vector<KeyFrame*> kf(nrows);
    std::map<KeyFrame*, int> row;
    for (int r = 0; r < nrows; r++) {
        Frame* F = empty_frame(V);
        frames.push_back(F);
        F->mBowVec = bow(off, word, val, r);
        kf[r] = new KeyFrame(*F, &map, &db);
        row[kf[r]] = r;
        kf[r]->mLoopScore = 0.f; kf[r]->mRelocScore = relocscore[r];
    }
    for (int r = 0; r < nrows; r++) {
        for (int c = 0; c < ncovis[r]; c++) kf[r]->mvpOrderedConnectedKeyFrames.push_back(kf[covis[10 * r + c]]);
        for (int c = conn_off[r]; c < conn_off[r + 1]; c++) kf[r]->mConnectedKeyFrameWeights[kf[conn[c]]] = 15;
    }
    for (int i = 0; i < nadd; i++) db.add(kf[add[i]]);
    for (int i = 0; i < nerase; i++) db.erase(kf[erase[i]]);
    double busy = 0.0;
    for (int q = 0; q < nq; q++) {
        std::vector<KeyFrame*> out;
        long unsigned int qid;
        Frame* F = nullptr;
        if (!loop) { F = empty_frame(V); frames.push_back(F); F->mBowVec = kf[query[q]]->mBowVec; }
        KeyFrame* Q = kf[query[q]];
        qid = 1000000 + q;                          // a fresh id: no keyframe carries it yet
        if (loop) Q->mnId = qid; else F->mnId = qid;
        const auto t0 = std::chrono::steady_clock::now();
        out = loop ? db.DetectLoopCandidates(Q, minscore[q]) : db.DetectRelocalizationCandidates(F);
        busy += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        ncand[q] = (int)out.size();
        for (size_t i = 0; i < out.size(); i++) cand[(size_t)q * nrows + i] = row[out[i]];
        for (int r = 0; r < nrows; r++) {
            const KeyFrame* K = kf[r];
            words[(size_t)q * nrows + r] = loop ? (K->mnLoopQuery == qid ? K->mnLoopWords : 0) : (K->mnRelocQuery == qid ? K->mnRelocWords : 0);
            score[(size_t)q * nrows + r] = loop ? K->mLoopScore : K->mRelocScore;
        }
    }
    if (seconds) *seconds = busy;
    for (KeyFrame* K : kf) delete K;
    for (Frame* F : frames) delete F;
}

}  // extern "C"
