// Interface between the tensor-core candidate pass (tc_eval.cu) and the evaluator (evaluator.cu).
#pragma once
#include "common.cuh"

namespace nrc {
namespace tc {

// Candidate lists produced by one pass: `nslots` lists per row (one per item segment), each ascending, `cap` entries long; cnt > cap marks an overflowed list.
struct CandLists {
    const int32_t* cand;   // [rows, nslots, cap]
    const int32_t* cnt;    // [rows, nslots]
    float* scratch;        // [rows, nslots, cap]: the candidates' approximate scores (the replay kernel overwrites
                           // them with exact ones)
    const float* margin;   // [rows] the per-user error margin the candidate kernel used
    int nslots, cap;
    int seg_items;         // items per segment: list s covers items [(s / CH) * seg_items, ...)
};

// bf16 copy of the item table + its largest row norm, kept in a library-owned buffer until the
// next call.  dim in {64, 128, 192, 256}.
int prepare_items(const float* V, int D, int N, cudaStream_t st);

// One tensor-core candidate pass over the prepared item table for the rows `users` (device ids).
// LQ = rank of the running threshold: every unmasked item whose score may exceed the LQ-th best
// score of the items before it IN ITS LIST'S ITEM SUBSET is reported, so each list is a superset
// of what a threshold over the whole prefix would keep:
//   pass 0 (main):   LQ = top_k + 1 -- every item of the exact top (K+1) is in some list;
//   pass 1 (replay): LQ = min(2*top_k, N) -- the lists hold every element that can enter the
//                    reference's heap (evaluate.h:38-41).
// Lists in slot order are ascending (slots are consecutive item ranges).
// Buffers are library-owned (one arena per pass) and reused between calls.
int run_pass(int pass, const float* U, const int32_t* users, int num_rows, const int64_t* train_ptr,
             const int32_t* train_idx, int LQ, int cap, CandLists* out, cudaStream_t st);

}  // namespace tc
}  // namespace nrc
