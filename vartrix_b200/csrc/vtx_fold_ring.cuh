// vtx_fold_ring.cuh -- how the warps of one vtx_k_sw_fold CTA take tiles and share the per-locus tables.
//
// The merged profile and the allele-column table of vtx_k_sw_fold depend only on the locus, and a deep locus has many
// tiles, so the warps of a CTA share one copy per locus in a ring of S slots instead of each building its own.
//
//   take     under the CTA's take lock: hand out the next tile of the CTA's current run with a ticket (its rank in
//            the CTA), or first claim a new run of consecutive tiles from the global cursor.  Tiles handed out by a
//            CTA only increase, so the loci in flight in a CTA are few and consecutive.  Nothing else is done under
//            the lock: one global atomic per run.
//   locate   outside any lock the warp finds its tile's locus, searching up from `hint`, the locus of a tile booked
//            earlier (a lower bound, because tiles and loci only increase).
//   book     in ticket order: either join the newest slot (it is tagged with this locus) or take a slot that no tile
//            is in flight on, tag it, clear its ready flag and become its builder.  Booking in ticket order means a
//            tile is counted in its slot before any later tile of the CTA can look for a free slot.
//   build    the builder fills the slot and publishes `ready` with release semantics; the other warps of that locus
//            wait for it with acquire semantics (and back off while they wait).
//   release  a warp drops its count on the slot after the last read of the slot's tables (after the allele pass and
//            its junction, not after the main pass).  A slot is reused only at count 0; its old locus can never get
//            another tile in this CTA then, because a newer locus has been booked.  A locus that comes back in the
//            newest slot after its count fell to 0 still finds its tables there; anywhere else it is rebuilt.
//
// Progress: every wait ends.
//   - The take lock is held for a bounded number of steps.  A warp that took a ticket locates (no waits) and books.
//   - Booking ticket q waits only for ticket q - 1 to be booked, and for a free slot.
//   - The oldest tile in flight in a CTA never waits on `ready`: its slot was built either by its own warp or by an
//     older tile's warp, which is no longer in flight.  So it finishes and releases its slot.  By induction every
//     booked tile finishes, which is all a booker waiting for a free slot needs: a warp releases its slot before it
//     takes another tile, so booked tiles in flight belong to other warps.
// There is no CTA-wide barrier after ring_init: a warp leaves as soon as a take finds the cursor past the last tile,
// which also covers grids with more warps than tiles.
//
// Everything here runs over an atomic policy `Sync` so that a CPU test drives the same code with std::thread workers
// (tests/fold_ring_rehearsal.cpp).  On the GPU one lane per warp takes, books, publishes and releases; the whole warp
// locates (fold_locate in vtx_sw_fold.cuh).
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define VTX_RING_FN __device__ __forceinline__
#else
#define VTX_RING_FN inline
#endif

namespace vtx {

constexpr uint32_t kFoldNoTile = 0xFFFFFFFFu;

// CTA-shared control state of a ring of S slots.  `lock`, `booked`, `hint`, `count` and `ready` are accessed atomically;
// the run state and `seq` only under the take lock, `newest` and `tag` only by the booking ticket holder, `mids` between
// publish and release.
template <int S> struct FoldRing {
    uint32_t lock;
    uint32_t run_next, run_end;      // tiles [run_next, run_end) of the CTA's current run are still to hand out
    uint32_t done;                   // the global cursor has passed the last tile
    uint32_t seq;                    // tickets handed out
    uint32_t booked;                 // tickets booked (the next ticket to book)
    uint32_t hint;                   // locus of the last booked tile
    uint32_t newest;                 // slot taken last
    uint32_t count[S];               // tiles in flight on the slot
    uint32_t ready[S];               // the slot's tables are built
    uint32_t tag[S];                 // locus the slot holds (kFoldNoTile: none yet)
    uint32_t mids[S];                // that locus's allele columns and shared extension: mid_ref | mid_alt << 8 | x << 16
};

struct FoldTake {
    uint32_t tile, ticket, hint;     // tile == kFoldNoTile: no tile left
};
struct FoldBook {
    uint32_t slot;
    bool build;                      // this warp builds the slot's tables
};

// tiles per run: at most kTileChunk per warp, fewer on small shards so that every CTA still gets >= ~16 runs (tail
// balance), never less than one
VTX_RING_FN uint32_t fold_run_len(uint32_t n_tiles, uint32_t ctas, uint32_t warps, uint32_t chunk)
{
    const uint32_t r = n_tiles / (ctas * 16u);
    return r < 1u ? 1u : r > warps * chunk ? warps * chunk : r;
}

template <int S> VTX_RING_FN void ring_init(FoldRing<S>& r)
{
    r.lock = 0; r.run_next = r.run_end = 0; r.done = 0; r.seq = r.booked = 0; r.hint = 0; r.newest = S - 1;
    for (int s = 0; s < S; ++s) { r.count[s] = 0; r.ready[s] = 0; r.tag[s] = kFoldNoTile; r.mids[s] = 0; }
}

// Hand out the CTA's next tile and its ticket (one caller per warp).
template <class Sync, int S>
VTX_RING_FN FoldTake ring_take(FoldRing<S>& r, uint32_t* cursor, uint32_t run_len, uint32_t n_tiles)
{
    FoldTake t{kFoldNoTile, 0, 0};
    while (!Sync::try_lock(&r.lock)) Sync::pause();
    if (r.run_next == r.run_end && !r.done) {
        const uint64_t b = uint64_t(Sync::grab(cursor)) * run_len;
        if (b >= n_tiles) {
            r.done = 1;
        } else {
            r.run_next = uint32_t(b);
            r.run_end = uint32_t(b + run_len < n_tiles ? b + run_len : n_tiles);
        }
    }
    if (r.run_next < r.run_end) {
        t.tile = r.run_next++;
        t.ticket = r.seq++;
        t.hint = Sync::load_relaxed(&r.hint);
    }
    Sync::unlock(&r.lock);
    return t;
}

// Count the taken tile in its locus's slot, in ticket order (one caller per warp, with the locus of t.tile).
template <class Sync, int S> VTX_RING_FN FoldBook ring_book(FoldRing<S>& r, uint32_t ticket, uint32_t locus)
{
    FoldBook b{0, false};
    while (Sync::load_acquire(&r.booked) != ticket) Sync::pause();
    if (r.tag[r.newest] == locus) {
        b.slot = r.newest;
        Sync::add(&r.count[b.slot], 1u);
    } else {
        uint32_t s = r.newest;
        for (;;) {                                              // oldest-first from the newest slot; the newest last
            s = s + 1 == uint32_t(S) ? 0 : s + 1;
            if (Sync::load_acquire(&r.count[s]) == 0) break;
            if (s == r.newest) Sync::pause();
        }
        r.tag[s] = locus;
        Sync::store_relaxed(&r.ready[s], 0u);
        Sync::add(&r.count[s], 1u);
        r.newest = b.slot = s;
        b.build = true;
    }
    Sync::store_relaxed(&r.hint, locus);
    Sync::store_release(&r.booked, ticket + 1);
    return b;
}

// the builder, after its tables and r.mids[slot] are written (and visible to the caller)
template <class Sync, int S> VTX_RING_FN void ring_publish(FoldRing<S>& r, uint32_t slot)
{
    Sync::store_release(&r.ready[slot], 1u);
}

template <class Sync, int S> VTX_RING_FN void ring_wait(FoldRing<S>& r, uint32_t slot)
{
    while (Sync::load_acquire(&r.ready[slot]) == 0) Sync::pause();
}

// after the last read of the slot's tables (by every lane of the warp)
template <class Sync, int S> VTX_RING_FN void ring_release(FoldRing<S>& r, uint32_t slot)
{
    Sync::sub_release(&r.count[slot], 1u);
}

}  // namespace vtx
