// frontend_ring.h — the batching ring shared by the front-ends (frontend.cpp: HTTP requests over gofr_batch_submit_slots;
// proto_frontend.cpp: gRPC messages over gofr_proto_batch_decode / _encode).
//
// Any number of caller threads hand in ONE record each and block until its result is ready; one dispatcher thread closes a
// batch when it is full or when its oldest record has waited max_wait_us, hands it to the front-end's `serve` and wakes
// the callers, each of which copies its own result out.  A small ring of batches rotates: while one is in flight the next
// fills, and a batch whose callers are slow to pick their results up (a descheduled thread) is skipped instead of
// stalling everybody.  What a record is, where its bytes are staged and how a batch is served belong to the front-end:
// this header knows batch numbers, slot numbers and arena byte ranges only.
//
// No lock on the call path (a mutex + condition variable version spent 5–10 µs per woken thread handing the mutex
// around: 93 k req/s at 256 threads):
//   claim     one CAS on the batch's claim word (closed bit | record count | arena bytes) reserves slot i and the arena
//             range [a, a + need); the record's bytes are copied in afterwards, outside any critical section (`filled`
//             counts them in).  Records therefore lie back to back in slot order.
//   close     the dispatcher sets the closed bit with fetch_or — the count is frozen at that instant
//   complete  the dispatcher publishes the round number in one futex word per group of 32 slots and wakes group 0;
//             the first thread of group g to notice wakes groups 2g+1 and 2g+2 (a wake tree: the dispatcher does not
//             pay one wake per thread)
//   recycle   the last caller to copy its result out reopens the batch
//
// Standard library and the futex system call only, so that the front-ends build against stub engines under ThreadSanitizer
// (tests/emu/frontend_stress.cpp, tests/emu/proto_frontend_stress.cpp).
#pragma once

#include <atomic>
#include <chrono>
#include <climits>
#include <cstdint>
#include <thread>
#include <time.h>

#include <linux/futex.h>
#include <sys/syscall.h>
#include <unistd.h>

namespace gofr_ring {

using Word = std::atomic<uint32_t>;
static_assert(sizeof(Word) == 4, "futex words are 32-bit");

inline void futex_wait(Word* w, uint32_t expect, const struct timespec* rel = nullptr) {
    syscall(SYS_futex, reinterpret_cast<uint32_t*>(w), FUTEX_WAIT_PRIVATE, expect, rel, nullptr, 0);
}
inline void futex_wake_all(Word* w) { syscall(SYS_futex, reinterpret_cast<uint32_t*>(w), FUTEX_WAKE_PRIVATE, INT_MAX, nullptr, nullptr, 0); }
inline void bump(Word* w) {
    w->fetch_add(1, std::memory_order_release);
    futex_wake_all(w);
}
inline int64_t mono_ns() {
    return std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

constexpr uint64_t kClosed = 1ull << 63;
inline uint32_t claim_count(uint64_t w) { return (uint32_t)(w >> 32) & 0x7FFFFFFFu; }
inline uint32_t claim_arena(uint64_t w) { return (uint32_t)w; }
constexpr uint32_t kGroup = 32;  // slots per wake word
constexpr int kBatches = 4;      // ring of batches

// The ring's side of one batch.  The front-end keeps its staging and outputs in an array of its own, indexed by the same
// batch number k.
struct Batch {
    std::atomic<uint64_t> claim{0};       // closed bit | count << 32 | arena bytes
    std::atomic<uint32_t> filled{0};      // records whose bytes are in place
    std::atomic<uint32_t> collected{0};   // callers that have copied their result out
    std::atomic<uint32_t> round{0};       // bumped at recycle; round r is complete when done[g] == r + 1
    std::atomic<int64_t> first_ns{0};     // arrival of the round's first record (0: not stored yet)
    uint32_t closed_count = 0;            // count at close (written by the dispatcher before done[] is published)
    int rc = 0;                           // what serve returned for the round
    Word* done = nullptr;                 // per group of kGroup slots: last completed round + 1
    Word* woke = nullptr;                 // per group: somebody already woke this group's children
};

// A caller's place in the ring: batch k, slot i, arena bytes from a, in round `round`.
struct Seat {
    int k;
    uint32_t i, a, round;
};

class Ring {
public:
    Ring(uint32_t max_batch_, uint32_t max_wait_us_)
        : max_batch(max_batch_), max_wait_us(max_wait_us_), groups((max_batch_ + kGroup - 1) / kGroup) {
        for (auto& x : b) {
            x.done = new Word[groups];
            x.woke = new Word[groups];
            for (uint32_t g = 0; g < groups; g++) { x.done[g].store(0); x.woke[g].store(0); }
        }
    }
    ~Ring() {
        stop();
        for (auto& x : b) { delete[] x.done; delete[] x.woke; }
    }
    Ring(const Ring&) = delete;
    Ring& operator=(const Ring&) = delete;

    // Starts the dispatcher.  serve(k, n, arena_bytes) runs batch k's n records, whose bytes take arena_bytes, and returns
    // the round's result code; the records' staging is complete when it is called.
    template <class Serve>
    void start(Serve serve) {
        worker = std::thread([this, serve]() mutable { dispatch(serve); });
    }
    // Callers already inside claim() leave it; no caller may be past claim() (the front-ends' destroy precondition).
    void stop() {
        stop_.store(true, std::memory_order_release);
        bump(&disp_seq);
        bump(&room_seq);
        if (worker.joinable()) worker.join();
    }

    // ---- the caller's side, in this order ----
    // Reserves a slot and `need` arena bytes in the filling batch; false once stop has begun.  The arena must hold max_batch
    // records of the largest `need` a caller passes: the count runs out first.
    bool claim(uint32_t need, Seat* s) {
        for (;;) {
            if (stop_.load(std::memory_order_acquire)) return false;
            const uint32_t rs = room_seq.load(std::memory_order_acquire);
            const int k = filling.load(std::memory_order_acquire);
            Batch& c = b[k];
            uint64_t w = c.claim.load(std::memory_order_acquire);
            if (!(w & kClosed) && claim_count(w) < max_batch) {
                if (!c.claim.compare_exchange_weak(w, w + (1ull << 32) + need, std::memory_order_acq_rel)) continue;
                s->k = k; s->i = claim_count(w); s->a = claim_arena(w);
                s->round = c.round.load(std::memory_order_acquire);  // stable until this caller has collected
                if (s->i == 0) c.first_ns.store(mono_ns(), std::memory_order_release);
                return true;
            }
            if (!(w & kClosed)) bump(&disp_seq);  // full: the dispatcher should close it now
            futex_wait(&room_seq, rs);            // until a batch is closed (the other one becomes current) or recycled
        }
    }
    // The record's bytes are in place.
    void filled(const Seat& s) {
        b[s.k].filled.fetch_add(1, std::memory_order_release);
        if (s.i == 0 || s.i + 1 == max_batch) bump(&disp_seq);  // start the round's timer / close a full batch
    }
    // Blocks until the round has been served, then passes the wake on; returns the batch's record count.  b[s.k].rc and the
    // front-end's outputs of slot s.i may be read until leave().
    uint32_t wait(const Seat& s) {
        Batch& x = b[s.k];
        const uint32_t g = s.i / kGroup;
        for (;;) {
            const uint32_t v = x.done[g].load(std::memory_order_acquire);
            if (v == s.round + 1) break;
            futex_wait(&x.done[g], v);
        }
        const uint32_t n = x.closed_count;
        const uint32_t g_used = (n + kGroup - 1) / kGroup;
        if (2 * g + 1 < g_used && x.woke[g].exchange(1, std::memory_order_acq_rel) == 0) {
            futex_wake_all(&x.done[2 * g + 1]);
            if (2 * g + 2 < g_used) futex_wake_all(&x.done[2 * g + 2]);
        }
        return n;
    }
    // The caller is done with its slot; the last one to leave reopens the batch.
    void leave(const Seat& s, uint32_t n) {
        Batch& x = b[s.k];
        if (x.collected.fetch_add(1, std::memory_order_acq_rel) + 1 == n) {
            const uint32_t g_used = (n + kGroup - 1) / kGroup;
            for (uint32_t k = 0; k < g_used; k++) x.woke[k].store(0, std::memory_order_relaxed);
            x.filled.store(0, std::memory_order_relaxed);
            x.collected.store(0, std::memory_order_relaxed);
            x.first_ns.store(0, std::memory_order_relaxed);
            x.round.store(s.round + 1, std::memory_order_release);
            x.claim.store(0, std::memory_order_release);
            bump(&room_seq);
            bump(&disp_seq);
        }
    }

    const uint32_t max_batch, max_wait_us, groups;
    Batch b[kBatches];
    std::atomic<uint64_t> batches{0}, records{0};
    // where the dispatcher's time goes, kept when debug is set before start()
    bool debug = false;
    int64_t dbg_spin_ns = 0, dbg_spin_max = 0, dbg_eng_ns = 0, dbg_eng_max = 0, dbg_wake_ns = 0, dbg_wake_max = 0;
    uint64_t dbg_eng_slow = 0;

private:
    template <class Serve>
    void dispatch(Serve& serve) {
        for (;;) {
            const uint32_t seq = disp_seq.load(std::memory_order_acquire);
            int k = filling.load(std::memory_order_relaxed);
            uint64_t w = b[k].claim.load(std::memory_order_acquire);
            if ((w & kClosed) || claim_count(w) == 0) {
                // Nothing to serve in the current batch.  Another one may hold records (a caller that read `filling` just
                // before a flip can claim a slot in a batch that was recycled in between); and if the current batch is
                // still handing out its previous round, any open batch is a better place for callers to go.
                int best = -1;
                for (int j = 1; j < kBatches && best < 0; j++) {
                    const uint64_t wj = b[(k + j) % kBatches].claim.load(std::memory_order_acquire);
                    if (!(wj & kClosed) && claim_count(wj) > 0) best = (k + j) % kBatches;
                }
                for (int j = 1; j < kBatches && best < 0 && (w & kClosed); j++)
                    if (!(b[(k + j) % kBatches].claim.load(std::memory_order_acquire) & kClosed)) best = (k + j) % kBatches;
                if (best >= 0) {
                    k = best;
                    filling.store(k, std::memory_order_release);
                    bump(&room_seq);
                    w = b[k].claim.load(std::memory_order_acquire);
                }
            }
            Batch& x = b[k];
            const bool stopping = stop_.load(std::memory_order_acquire);
            if ((w & kClosed) || claim_count(w) == 0) {  // still being collected by its previous round / nothing to do
                if (stopping && !(w & kClosed)) return;
                futex_wait(&disp_seq, seq);
                continue;
            }
            if (claim_count(w) < max_batch && !stopping) {
                // not full: wait until the oldest record has been here max_wait_us (or the batch fills up)
                const int64_t first = x.first_ns.load(std::memory_order_acquire), now = mono_ns();
                const int64_t deadline = (first ? first : now) + (int64_t)max_wait_us * 1000;
                if (now < deadline) {
                    struct timespec rel;
                    rel.tv_sec = (deadline - now) / 1000000000;
                    rel.tv_nsec = (deadline - now) % 1000000000;
                    futex_wait(&disp_seq, seq, &rel);
                    continue;
                }
            }
            // close: the count is frozen by the fetch_or; callers move on to the next open batch of the ring
            w = x.claim.fetch_or(kClosed, std::memory_order_acq_rel);
            const uint32_t n = claim_count(w);
            x.closed_count = n;
            int next = (k + 1) % kBatches;
            for (int j = 1; j < kBatches; j++)
                if (!(b[(k + j) % kBatches].claim.load(std::memory_order_acquire) & kClosed)) { next = (k + j) % kBatches; break; }
            filling.store(next, std::memory_order_release);
            bump(&room_seq);
            const int64_t t_close = debug ? mono_ns() : 0;
            while (x.filled.load(std::memory_order_acquire) != n) {  // the last claimants are still copying their bytes in
#if defined(__x86_64__)
                __builtin_ia32_pause();
#endif
            }
            const int64_t t_filled = debug ? mono_ns() : 0;
            x.rc = serve(k, n, claim_arena(w));
            const int64_t t_eng = debug ? mono_ns() : 0;
            batches.fetch_add(1, std::memory_order_relaxed);
            records.fetch_add(n, std::memory_order_relaxed);
            // publish the round in every group's word, then start the wake tree at its root.  DESCENDING group order: a
            // caller of group g that is already awake may see done[g] == r1 at any moment and wake its children 2g+1 and
            // 2g+2 exactly once (woke[g]); with release stores from the highest group down, seeing done[g] implies both
            // children's words are already stored, so a child woken by that futex_wake cannot read the old value and go
            // back to sleep with nobody left to wake it.
            const uint32_t r1 = x.round.load(std::memory_order_relaxed) + 1, g_used = (n + kGroup - 1) / kGroup;
            for (uint32_t g = g_used; g-- > 0;) x.done[g].store(r1, std::memory_order_release);
            futex_wake_all(&x.done[0]);
            if (debug) {
                const int64_t t_end = mono_ns();
                dbg_spin_ns += t_filled - t_close; if (t_filled - t_close > dbg_spin_max) dbg_spin_max = t_filled - t_close;
                dbg_eng_ns += t_eng - t_filled; if (t_eng - t_filled > dbg_eng_max) dbg_eng_max = t_eng - t_filled;
                if (t_eng - t_filled > 5000000) dbg_eng_slow++;
                dbg_wake_ns += t_end - t_eng; if (t_end - t_eng > dbg_wake_max) dbg_wake_max = t_end - t_eng;
            }
        }
    }

    std::atomic<int> filling{0};          // the batch callers try first
    std::atomic<bool> stop_{false};
    Word disp_seq{0};                     // dispatcher sleeps on this: first claim of a round, full batch, recycle, stop
    Word room_seq{0};                     // callers without a slot sleep on this: batch closed (flip) or recycled
    std::thread worker;
};

}  // namespace gofr_ring
