// tests/simt/simt_runtime.cpp -- TEST INFRASTRUCTURE: scheduler of the SIMT interpreter (see cuda_runtime.h here).
//
// One launch = blocks executed one after another; one block = one fiber (ucontext) per CUDA thread, resumed
// round robin.  A fiber runs until it reaches a point where it has to wait for other threads (block barrier, warp
// collective, mbarrier wait); a full round in which no thread gets anywhere is reported as a deadlock.
#include <cuda_runtime.h>

#include <ucontext.h>

#include <map>
#include <vector>

#if defined(__SANITIZE_ADDRESS__)
#include <sanitizer/asan_interface.h>
#endif

#include "crt_ptx.cuh"

namespace crt { // the kernels' dynamic shared-memory arrays ("extern __shared__ T name[]")
__attribute__((aligned(128))) unsigned char smem_raw[232448];
__attribute__((aligned(128))) unsigned heads[232448 / 4];
__attribute__((aligned(128))) unsigned char vsm[232448];
} // namespace crt

namespace simt {

Thread *g_cur = nullptr;
unsigned char *g_smem_anchor = crt::smem_raw;
long g_launches = 0, g_blocks = 0;

namespace {

constexpr size_t kStack = 256 * 1024;

struct Copy { void *dst; const void *src; unsigned bytes; };

struct Fiber {
    Thread t;
    ucontext_t ctx;
    unsigned char *stack = nullptr;
    bool done = false;
    std::vector<std::vector<Copy>> lane_groups;  // cp.async: committed groups, oldest first
    std::vector<Copy> lane_open;
    std::vector<std::vector<Copy>> store_groups; // bulk stores: committed groups, oldest first
    std::vector<Copy> store_open;
};

} // namespace

struct Warp {
    unsigned arrived = 0, exited = 0, cur_mask = 0, gen = 0, members = 0;
    uint64_t buf[2][32];
};

namespace {

struct Block {
    std::vector<Fiber> fibers;
    std::vector<Warp> warps;
    int nthreads = 0, exited = 0;
    int bar_arrived = 0, bar_or[2] = { 0, 0 };
    unsigned bar_gen = 0;
    std::map<uint64_t *, std::vector<Copy>> pending_loads; // per mbarrier
    const std::function<void()> *body = nullptr;
};

Block *g_block = nullptr;
Fiber *g_fiber = nullptr;
ucontext_t g_sched;
unsigned long g_progress = 0;

[[noreturn]] void fatal(const char *what)
{
    if (g_cur)
        fprintf(stderr, "simt: %s (block %u,%u thread %u)\n", what, g_cur->bid.x, g_cur->bid.y, g_cur->tid.x);
    else
        fprintf(stderr, "simt: %s\n", what);
    abort();
}

void do_copy(const Copy &c) { memcpy(c.dst, c.src, c.bytes); }

void warp_try_release(Warp &w)
{
    if (w.arrived && (((w.arrived | w.exited) & w.cur_mask & w.members) == (w.cur_mask & w.members))) {
        w.arrived = 0;
        w.gen++;
        g_progress++;
    }
}

void block_try_release(Block &b)
{
    if (b.bar_arrived && b.bar_arrived + b.exited == b.nthreads) {
        b.bar_arrived = 0;
        b.bar_or[(b.bar_gen + 1) & 1] = 0;
        b.bar_gen++;
        g_progress++;
    }
}

void fiber_entry()
{
    Fiber *f = g_fiber;
    (*g_block->body)();
    // what the hardware would still complete after the thread's last instruction
    for (auto &g : f->lane_groups) for (auto &c : g) do_copy(c);
    for (auto &c : f->lane_open) do_copy(c);
    for (auto &g : f->store_groups) for (auto &c : g) do_copy(c);
    for (auto &c : f->store_open) do_copy(c);
    f->done = true;
    g_block->exited++;
    f->t.warp->exited |= 1u << f->t.lane;
    warp_try_release(*f->t.warp);
    block_try_release(*g_block);
    g_progress++;
    swapcontext(&f->ctx, &g_sched);
    fatal("resumed a finished thread");
}

} // namespace

void yield_blocked() { swapcontext(&g_fiber->ctx, &g_sched); }
void note_progress() { g_progress++; }

void block_barrier(int pred, int *any)
{
    Block &b = *g_block;
    const unsigned gen = b.bar_gen;
    if (pred) b.bar_or[gen & 1] = 1;
    b.bar_arrived++;
    g_progress++;
    block_try_release(b);
    while (b.bar_gen == gen) yield_blocked();
    if (any) *any = b.bar_or[gen & 1];
}

const uint64_t *warp_exchange(unsigned mask, uint64_t v)
{
    Thread *t = g_cur;
    Warp &w = *t->warp;
    if (!((mask >> t->lane) & 1u)) fatal("warp collective: calling lane is not in its own mask");
    const unsigned gen = w.gen;
    if (w.arrived == 0) w.cur_mask = mask;
    else if (w.cur_mask != mask) fatal("warp collective: lanes of one warp disagree on the mask (divergent collectives)");
    w.buf[gen & 1][t->lane] = v;
    w.arrived |= 1u << t->lane;
    g_progress++;
    warp_try_release(w);
    while (w.gen == gen) yield_blocked();
    return w.buf[gen & 1];
}

void ptx_fail(const char *what) { fatal(what); }

// ---- mbarrier: [phase:1][pending:15][init:15] in the low word, signed tx-count in the high word
namespace {
struct Mbar { unsigned phase, pending, init; int tx; };
Mbar mb_get(const uint64_t *bar)
{
    const uint64_t v = *bar;
    Mbar m;
    m.phase = (unsigned) (v & 1u);
    m.pending = (unsigned) ((v >> 1) & 0x7fffu);
    m.init = (unsigned) ((v >> 16) & 0x7fffu);
    m.tx = (int) (uint32_t) (v >> 32);
    return m;
}
void mb_put(uint64_t *bar, const Mbar &m)
{
    *bar = (uint64_t) m.phase | ((uint64_t) m.pending << 1) | ((uint64_t) m.init << 16) | ((uint64_t) (uint32_t) m.tx << 32);
}
void mb_complete_if_done(Mbar &m)
{
    if (m.pending == 0 && m.tx == 0) {
        m.phase ^= 1u;
        m.pending = m.init;
        g_progress++;
    }
}
} // namespace

void mbar_init(uint64_t *bar, unsigned count)
{
    if ((uintptr_t) bar & 7) fatal("mbarrier.init: misaligned barrier");
    Mbar m = { 0u, count, count, 0 };
    mb_put(bar, m);
    g_block->pending_loads[bar].clear();
}

void mbar_expect_tx(uint64_t *bar, unsigned bytes)
{
    Mbar m = mb_get(bar);
    if (m.init == 0) fatal("mbarrier.arrive.expect_tx on an uninitialised barrier");
    if (m.pending == 0) fatal("mbarrier.arrive: more arrivals than the barrier was initialised for");
    m.tx += (int) bytes;
    m.pending -= 1;
    mb_complete_if_done(m);
    mb_put(bar, m);
}

void bulk_load(void *dst, const void *src, unsigned bytes, uint64_t *bar)
{
    if (((uintptr_t) dst & 15) || ((uintptr_t) src & 15) || (bytes & 15) || bytes == 0)
        fatal("cp.async.bulk (global -> shared): dst, src and size must be multiples of 16");
    g_block->pending_loads[bar].push_back(Copy{ dst, src, bytes });
}

void mbar_wait(uint64_t *bar, unsigned parity)
{
    for (;;) {
        Mbar m = mb_get(bar);
        if (m.init == 0) fatal("mbarrier.try_wait on an uninitialised barrier");
        std::vector<Copy> &q = g_block->pending_loads[bar];
        if (!q.empty()) { // the copies land now, at the last possible moment
            for (auto &c : q) {
                do_copy(c);
                m.tx -= (int) c.bytes;
            }
            q.clear();
            mb_complete_if_done(m);
            mb_put(bar, m);
        }
        if (m.phase != (parity & 1u)) break;
        yield_blocked();
    }
    g_progress++;
}

void lane_copy16(void *dst, const void *src)
{
    if (((uintptr_t) dst & 15) || ((uintptr_t) src & 15)) fatal("cp.async 16: misaligned address");
    g_fiber->lane_open.push_back(Copy{ dst, src, 16u });
}
void lane_commit()
{
    g_fiber->lane_groups.push_back(g_fiber->lane_open);
    g_fiber->lane_open.clear();
}
void lane_wait(int pending)
{
    auto &g = g_fiber->lane_groups;
    while ((int) g.size() > pending) {
        for (auto &c : g.front()) do_copy(c);
        g.erase(g.begin());
    }
}

void bulk_store(void *dst, const void *src, unsigned bytes)
{
    if (((uintptr_t) dst & 15) || ((uintptr_t) src & 15) || (bytes & 15) || bytes == 0)
        fatal("cp.async.bulk (shared -> global): dst, src and size must be multiples of 16");
    g_fiber->store_open.push_back(Copy{ dst, src, bytes });
}
void bulk_store_commit()
{
    g_fiber->store_groups.push_back(g_fiber->store_open);
    g_fiber->store_open.clear();
}
void bulk_store_wait_read(int pending)
{
    auto &g = g_fiber->store_groups;
    while ((int) g.size() > pending) {
        for (auto &c : g.front()) do_copy(c);
        g.erase(g.begin());
    }
}

// ---- device memory: plain host memory, filled with a pattern (cudaMalloc does not zero either)
void *dev_alloc(size_t bytes)
{
    // cudaMalloc hands out 256-byte granular blocks, and the kernels rely on being allowed to read up to the next
    // 16-byte boundary past an image (include/crtx_batch.h).  SIMT_TIGHT_ALLOC=1 (with an AddressSanitizer build of
    // the interpreter, see build.py) grants exactly that and nothing more, so any other over-read is reported.
    static int tight = -1;
    if (tight < 0) {
        const char *e = getenv("SIMT_TIGHT_ALLOC");
        tight = (e && *e == '1') ? 1 : 0;
    }
    void *p = nullptr;
    const size_t gran = tight ? 16 : 256;
    const size_t n = ((bytes ? bytes : 1) + gran - 1) & ~(gran - 1);
    if (posix_memalign(&p, 256, n + (tight ? 0 : 256))) return nullptr;
    memset(p, 0xcd, n + (tight ? 0 : 256));
    return p;
}
void dev_free(void *p) { free(p); }

void launch(dim3 grid, dim3 block, size_t smem_bytes, const std::function<void()> &body)
{
    if (g_cur) fatal("nested launch");
    const int nthreads = (int) (block.x * block.y * block.z);
    if (nthreads <= 0 || nthreads > 1024) fatal("launch: bad block size");
    if (smem_bytes > sizeof(crt::smem_raw)) fatal("launch: dynamic shared memory above 227 KB");
    g_launches++;
    static std::vector<unsigned char *> stacks;
    while ((int) stacks.size() < nthreads) {
        void *s = nullptr;
        if (posix_memalign(&s, 4096, kStack)) fatal("out of memory (fiber stacks)");
        stacks.push_back((unsigned char *) s);
    }
    // Blocks of a launch may run in any order, or together: SIMT_BLOCKS=reverse runs them last to first, which turns a
    // hidden "a later block reads what an earlier one wrote" dependence into a wrong result.
    static int block_order = -1;
    if (block_order < 0) {
        const char *e = getenv("SIMT_BLOCKS");
        block_order = (e && !strncmp(e, "reverse", 7)) ? 1 : 0;
    }
    const unsigned long long nblocks = (unsigned long long) grid.x * grid.y * grid.z;
    for (unsigned long long bi = 0; bi < nblocks; bi++) {
        const unsigned long long lin = block_order ? nblocks - 1 - bi : bi;
        const unsigned bx = (unsigned) (lin % grid.x), by = (unsigned) ((lin / grid.x) % grid.y), bz = (unsigned) (lin / ((unsigned long long) grid.x * grid.y));
        g_blocks++;
        Block blk;
        blk.nthreads = nthreads;
        blk.body = &body;
        blk.fibers.resize(nthreads);
        blk.warps.resize((nthreads + 31) / 32);
#if defined(__SANITIZE_ADDRESS__)
        ASAN_UNPOISON_MEMORY_REGION(crt::smem_raw, sizeof(crt::smem_raw));
        ASAN_UNPOISON_MEMORY_REGION(crt::heads, sizeof(crt::heads));
        ASAN_UNPOISON_MEMORY_REGION(crt::vsm, sizeof(crt::vsm));
#endif
        memset(crt::smem_raw, 0xa5, sizeof(crt::smem_raw)); // shared memory starts out as garbage
        memset(crt::heads, 0xa5, sizeof(crt::heads));
        memset(crt::vsm, 0xa5, sizeof(crt::vsm));
#if defined(__SANITIZE_ADDRESS__)
        { // only the dynamic shared memory the launch asked for exists (the three arrays are the same window by name)
            const size_t used = (smem_bytes + 7) & ~(size_t) 7;
            ASAN_POISON_MEMORY_REGION(crt::smem_raw + used, sizeof(crt::smem_raw) - used);
            ASAN_POISON_MEMORY_REGION(reinterpret_cast<unsigned char *>(crt::heads) + used, sizeof(crt::heads) - used);
            ASAN_POISON_MEMORY_REGION(crt::vsm + used, sizeof(crt::vsm) - used);
        }
#endif
        g_block = &blk;
        for (int i = 0; i < nthreads; i++) {
            Fiber &f = blk.fibers[i];
            f.t.tid.x = (unsigned) i % block.x;
            f.t.tid.y = ((unsigned) i / block.x) % block.y;
            f.t.tid.z = (unsigned) i / (block.x * block.y);
            f.t.bid.x = bx; f.t.bid.y = by; f.t.bid.z = bz;
            f.t.bdim = block;
            f.t.gdim = grid;
            f.t.lin = i;
            f.t.lane = i & 31;
            f.t.warp = &blk.warps[i >> 5];
            blk.warps[i >> 5].members |= 1u << (i & 31);
            f.stack = stacks[i];
            getcontext(&f.ctx);
            f.ctx.uc_stack.ss_sp = f.stack;
            f.ctx.uc_stack.ss_size = kStack;
            f.ctx.uc_link = nullptr;
            makecontext(&f.ctx, (void (*)()) fiber_entry, 0);
        }
        // Order in which runnable threads are resumed within a round.  Any order is a legal interleaving of a CUDA
        // block; SIMT_SCHEDULE=reverse or random[:seed] (reshuffled every round) re-runs a test under other ones, which
        // is how an accidental dependence on "lower threads run first" shows up without a GPU.
        static int mode = -1;
        static unsigned long long rng = 0x9e3779b97f4a7c15ull;
        if (mode < 0) {
            const char *e = getenv("SIMT_SCHEDULE");
            mode = 0;
            if (e && !strncmp(e, "reverse", 7)) mode = 1;
            if (e && !strncmp(e, "random", 6)) {
                mode = 2;
                if (e[6] == ':') rng ^= strtoull(e + 7, nullptr, 10) * 0xd1342543de82ef95ull;
            }
        }
        std::vector<int> order(nthreads);
        for (int i = 0; i < nthreads; i++) order[i] = (mode == 1) ? nthreads - 1 - i : i;
        int live = nthreads;
        while (live > 0) {
            const unsigned long before = g_progress;
            if (mode == 2) {
                for (int i = nthreads - 1; i > 0; i--) {
                    rng = rng * 6364136223846793005ull + 1442695040888963407ull;
                    const int j = (int) ((rng >> 33) % (unsigned) (i + 1));
                    const int t = order[i]; order[i] = order[j]; order[j] = t;
                }
            }
            for (int oi = 0; oi < nthreads; oi++) {
                const int i = order[oi];
                Fiber &f = blk.fibers[i];
                if (f.done) continue;
                g_fiber = &f;
                g_cur = &f.t;
                swapcontext(&g_sched, &f.ctx);
                if (f.done) live--;
            }
            g_cur = nullptr;
            if (live > 0 && g_progress == before) {
                fprintf(stderr, "simt: deadlock in block (%u,%u): %d threads wait for something that cannot happen\n", bx, by, live);
                abort();
            }
        }
        g_block = nullptr;
        g_fiber = nullptr;
    }
}

} // namespace simt

extern "C" long simt_launches(void) { return simt::g_launches; }
extern "C" long simt_blocks(void) { return simt::g_blocks; }
