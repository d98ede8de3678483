// Packing of calls into one-wave groups, the protocol of both engines (api.cu: consensus, readlevel.cu: read-level).
// Plain C++ without CUDA, so that a CPU test can drive it with a fake engine (tests/test_packing.py).  A call's windows
// go into the open group window by window: a call that does not fit what is left of it is split (windows are
// independent, medaka/prediction.py:40-52), so every group of a long run is full however the caller sized its calls.
// The engine supplies, each returning MDK_OK (0) or an error code that the core passes on:
//   open(windows)        make buffers ready for a group of up to `windows` windows
//   capacity(len)        windows of length len the current buffers hold (int64_t)
//   stage(first, n, at)  windows [first, first + n) of the call into the open group from window `at` on
//   launch()             run the group and copy its results back
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

namespace mdk {

struct Packing {
    struct Piece {                 // one call's share of a group
        float *probs, *logits;     // the call's outputs ([B][len][5] probabilities; logits and labels may be null)
        uint8_t *labels;
        int64_t first, n;          // first window in the call, windows
        uint8_t *quals;            // [B][len] phred bytes of the argmax class, or null (then probs may be null too:
                                   // a decoded call, mdk_engine_submit_decoded, wants labels and quals only)
        const uint8_t *ref;        // a variant-decoded call (mdk_engine_submit_variant_decoded): its [B][len] reference
        float *pred_q, *ref_q;     // bytes, and its phreds; `labels` then receives the call bytes.  Null otherwise.
    };
    std::vector<Piece> pieces;     // of the open group, or of the group last launched
    int64_t windows = 0, len = 0;  // the group's windows so far and its window length
    bool open = false;
    int64_t serial = -1;           // serial number of the open or last opened group
    int64_t launched = -1;         // serial number of the last launched group
    static constexpr int TICKET_RING = 4096;
    int64_t ticket_group[TICKET_RING] = {};   // ticket -> group serial, for the last TICKET_RING tickets
    int64_t tickets = 0;

    template <class Eng>
    int launch(Eng &&eng) {     // seal the open group and run it
        if (!open) return 0;
        open = false;
        if (pieces.empty()) return 0;
        const int rc = eng.launch();
        if (!rc) launched = serial;
        return rc;
    }

    // One call of B windows of length L, with at most gmax windows to a group; ticket may be null.
    template <class Eng>
    int enqueue(Eng &&eng, int64_t B, int64_t L, float *probs, float *logits, uint8_t *labels, int64_t gmax,
                int64_t *ticket, uint8_t *quals = nullptr, const uint8_t *ref = nullptr, float *pred_q = nullptr,
                float *ref_q = nullptr) {
        int rc;
        if (open && len != L && (rc = launch(eng))) return rc;      // a new window length seals the open group
        for (int64_t done = 0; done < B;) {
            if (!open) {
                if ((rc = eng.open(std::min(B - done, gmax)))) return rc;
                pieces.clear();
                windows = 0; len = L;
                open = true;
                serial++;
            }
            int64_t room = std::min(gmax, eng.capacity(L)) - windows;
            if (windows == 0) room = std::max<int64_t>(room, 1);  // a fresh group takes one window at least
            if (room < 1) {
                if ((rc = launch(eng))) return rc;
                continue;
            }
            const int64_t n = std::min(room, B - done);
            if ((rc = eng.stage(done, n, windows))) return rc;
            pieces.push_back(Piece{probs, logits, labels, done, n, quals, ref, pred_q, ref_q});
            windows += n;
            done += n;
            if (done == B && ticket) {                                  // the piece that ends the call
                ticket_group[tickets % TICKET_RING] = serial;
                *ticket = tickets++;
            }
            if (n == room && (rc = launch(eng))) return rc;             // full: launch at once
        }
        return 0;
    }

    // The group a wait on ticket (< tickets) must see complete, launched if still open.  A ticket older than the ring
    // takes the oldest ticket's group the ring holds: serials grow with tickets, so that is its own group or a later one.
    template <class Eng>
    int settle(Eng &&eng, int64_t ticket, int64_t *group) {
        *group = ticket_group[std::max(ticket, tickets - TICKET_RING) % TICKET_RING];
        return open && *group == serial ? launch(eng) : 0;
    }
};

}  // namespace mdk
