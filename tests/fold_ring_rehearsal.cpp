// Drives the tile hand-out and slot ring of vtx_k_sw_fold (vartrix_b200/csrc/vtx_fold_ring.cuh) with std::thread
// workers in place of warps: the same take / book / publish / wait / release functions, over std::atomic_ref.
//   fold_ring_rehearsal <mode> <seed>     mode: ones | huge | mixed | sparse
// For every S in 1..13 and several CTA shapes it checks that every tile is handed out exactly once, with the locus it
// belongs to, that a worker only reads a slot holding its locus's finished tables (also while other workers rebuild
// slots), and that every run ends (the caller's timeout).  Built with -fsanitize=thread where the toolchain has it.
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../vartrix_b200/csrc/vtx_fold_ring.cuh"

using namespace vtx;

struct HostSync {
    using ref = std::atomic_ref<uint32_t>;
    static bool try_lock(uint32_t* p)
    {
        uint32_t z = 0;
        return ref(*p).compare_exchange_strong(z, 1u, std::memory_order_acquire, std::memory_order_relaxed);
    }
    static void unlock(uint32_t* p) { ref(*p).store(0u, std::memory_order_release); }
    static uint32_t grab(uint32_t* cursor) { return ref(*cursor).fetch_add(1u, std::memory_order_relaxed); }
    static uint32_t load_relaxed(uint32_t* p) { return ref(*p).load(std::memory_order_relaxed); }
    static uint32_t load_acquire(uint32_t* p) { return ref(*p).load(std::memory_order_acquire); }
    static void store_relaxed(uint32_t* p, uint32_t v) { ref(*p).store(v, std::memory_order_relaxed); }
    static void store_release(uint32_t* p, uint32_t v) { ref(*p).store(v, std::memory_order_release); }
    static void add(uint32_t* p, uint32_t v) { ref(*p).fetch_add(v, std::memory_order_relaxed); }
    static void sub_release(uint32_t* p, uint32_t v) { ref(*p).fetch_sub(v, std::memory_order_release); }
    static void pause() { std::this_thread::yield(); }
};

constexpr int kWords = 8;                       // stand-in for a slot's tables: word k of locus l holds l * 8 + k

static uint64_t next(uint64_t& x)
{
    x ^= x << 13; x ^= x >> 7; x ^= x << 17;
    return x;
}

static std::atomic<int> g_errors{0};
static void fail(const char* what, uint32_t a, uint32_t b)
{
    if (g_errors.fetch_add(1) < 10) std::fprintf(stderr, "FAIL %s (%u, %u)\n", what, a, b);
}

template <int S> struct Cta {
    FoldRing<S> ring;
    uint32_t table[S][kWords];                  // plain memory: ordering comes from the ring alone
};

template <int S>
static void worker(Cta<S>* cta, uint32_t* cursor, uint32_t run_len, const std::vector<uint32_t>* ts,
                   std::atomic<uint32_t>* handed, uint64_t seed)
{
    const uint32_t n_loci = uint32_t(ts->size() - 1), n_tiles = ts->back();
    uint64_t x = seed | 1;
    uint32_t last = 0;
    bool first = true;
    for (;;) {
        const FoldTake tk = ring_take<HostSync>(cta->ring, cursor, run_len, n_tiles);
        if (tk.tile == kFoldNoTile) break;
        // the locus, walking up from the hint: a hint past the tile's locus gives a wrong locus below
        uint32_t l = tk.hint;
        while (l + 1 < n_loci && (*ts)[l + 1] <= tk.tile) ++l;
        if (next(x) % 3 == 0) std::this_thread::yield();
        const FoldBook bk = ring_book<HostSync>(cta->ring, tk.ticket, l);
        const struct { uint32_t tile, locus, slot; bool build; } c{tk.tile, l, bk.slot, bk.build};
        if (c.tile >= n_tiles) { fail("tile out of range", c.tile, n_tiles); break; }
        handed[c.tile].fetch_add(1, std::memory_order_relaxed);
        if (!first && c.tile <= last) fail("tiles of a worker not increasing", last, c.tile);
        first = false; last = c.tile;
        if (c.locus >= n_loci || !((*ts)[c.locus] <= c.tile && c.tile < (*ts)[c.locus + 1])) fail("wrong locus", c.tile, c.locus);
        if (c.slot >= uint32_t(S)) { fail("slot out of range", c.slot, S); break; }
        uint32_t* t = cta->table[c.slot];
        if (c.build) {
            for (int k = 0; k < kWords; ++k) {
                t[k] = c.locus * kWords + k;
                if (next(x) % 4 == 0) std::this_thread::yield();
            }
            cta->ring.mids[c.slot] = c.locus;
            ring_publish<HostSync>(cta->ring, c.slot);
        } else {
            ring_wait<HostSync>(cta->ring, c.slot);
        }
        // "the tile": read the tables twice with a pause in between; the slot must hold this locus throughout
        for (int pass = 0; pass < 2; ++pass) {
            if (cta->ring.mids[c.slot] != c.locus) fail("slot header of another locus", c.locus, cta->ring.mids[c.slot]);
            for (int k = 0; k < kWords; ++k)
                if (t[k] != c.locus * kWords + k) { fail("slot table of another locus", c.locus, t[k]); break; }
            if (next(x) % 2 == 0) std::this_thread::yield();
        }
        ring_release<HostSync>(cta->ring, c.slot);
    }
}

template <int S> static int run(const std::vector<uint32_t>& ts, int ctas, int workers, uint64_t seed)
{
    const uint32_t n_tiles = ts.back();
    std::vector<Cta<S>> cta(ctas);
    for (auto& c : cta) {
        ring_init(c.ring);
        std::memset(c.table, 0xFF, sizeof c.table);
    }
    // the kernel's run length, and for variety sometimes a single tile or a run of several per worker
    uint32_t run_len = fold_run_len(n_tiles, ctas, workers, 8);
    if (seed % 3 == 1) run_len = 1;
    if (seed % 3 == 2) run_len = uint32_t(workers) * 3 + 1;
    uint32_t cursor = 0;
    std::vector<std::atomic<uint32_t>> handed(n_tiles);
    for (auto& h : handed) h.store(0);
    std::vector<std::thread> th;
    for (int c = 0; c < ctas; ++c)
        for (int w = 0; w < workers; ++w)
            th.emplace_back(worker<S>, &cta[c], &cursor, run_len, &ts, handed.data(), seed * 1000003 + c * 64 + w);
    for (auto& t : th) t.join();
    for (uint32_t i = 0; i < n_tiles; ++i)
        if (handed[i].load() != 1) { fail("tile not handed out exactly once", i, handed[i].load()); break; }
    for (auto& c : cta)
        for (int s = 0; s < S; ++s)
            if (c.ring.count[s] != 0) fail("slot count left over", s, c.ring.count[s]);
    return g_errors.load();
}

template <int S> static int run_s(int s, const std::vector<uint32_t>& ts, int ctas, int workers, uint64_t seed)
{
    if constexpr (S > 13) return -1;
    else return s == S ? run<S>(ts, ctas, workers, seed) : run_s<S + 1>(s, ts, ctas, workers, seed);
}

static std::vector<uint32_t> make_tiles(const std::string& mode, uint64_t& x)
{
    std::vector<uint32_t> cnt;
    if (mode == "ones") {                       // depth <= 4: every locus one tile
        cnt.assign(600 + next(x) % 200, 1);
    } else if (mode == "huge") {                // one deep locus among shallow ones
        for (int i = 0; i < 40; ++i) cnt.push_back(1 + next(x) % 3);
        cnt.push_back(2500 + next(x) % 500);
        for (int i = 0; i < 40; ++i) cnt.push_back(1 + next(x) % 3);
    } else if (mode == "mixed") {               // any depth, loci without tiles in between
        for (int i = 0; i < 250; ++i) cnt.push_back(next(x) % 4 == 0 ? 0 : 1 + next(x) % 24);
    } else {                                    // sparse: long runs of loci without tiles, tiny totals
        const int n = 1 + int(next(x) % 40);
        for (int i = 0; i < n; ++i) {
            for (uint64_t z = next(x) % 50; z; --z) cnt.push_back(0);
            cnt.push_back(1 + next(x) % 2);
        }
        for (uint64_t z = next(x) % 5; z; --z) cnt.push_back(0);
    }
    std::vector<uint32_t> ts(1, 0);
    for (uint32_t c : cnt) ts.push_back(ts.back() + c);
    return ts;
}

int main(int argc, char** argv)
{
    if (argc < 3) { std::fprintf(stderr, "usage: %s ones|huge|mixed|sparse seed\n", argv[0]); return 2; }
    const std::string mode = argv[1];
    uint64_t x = std::strtoull(argv[2], nullptr, 10) * 0x9E3779B97F4A7C15ull + 1;
    const int shapes[][2] = {{1, 1}, {1, 13}, {2, 5}, {3, 18}, {2, 20}};   // (CTAs, workers per CTA)
    int runs = 0;
    for (int s = 1; s <= 13; ++s)
        for (const auto& sh : shapes) {
            const std::vector<uint32_t> ts = make_tiles(mode, x);
            if (run_s<1>(s, ts, sh[0], sh[1], next(x)) != 0) {
                std::fprintf(stderr, "mode %s S %d CTAs %d workers %d tiles %u\n", mode.c_str(), s, sh[0], sh[1], ts.back());
                return 1;
            }
            ++runs;
        }
    std::printf("ok %d runs\n", runs);
    return 0;
}
