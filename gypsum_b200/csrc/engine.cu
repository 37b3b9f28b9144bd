// C ABI of the engine (include/gypsum_b200.h): owns device memory, builds launch plans, drives the kernels.  This file
// holds the engine's lifetime, its IQ and every acquisition entry point; receiver.cu holds the trackers.
// Host side of the reference path it replaces: gypsum/acquisition.py:154-219 (the per-bin scan and its memo
// wrapper) and gypsum/utils.py:77-108.
#include <cmath>
#include <cstdlib>
#include <map>
#include <numeric>

#include "host.cuh"

using namespace gb;
using namespace gb::capi;

static_assert(sizeof(gb200_cell_record) == sizeof(CellRecord), "ABI record and device record must match");
static_assert(sizeof(gb200_best_record) == sizeof(BestRecord), "ABI best record and device record must match");

// A pipelined stream of grid batches: slot k's host->device copy, compute and device->host copy run on three streams.
struct gb200_grid_stream {
    gb200_engine* e = nullptr;
    int n_blocks = 0, M = 0, P = 0, D = 0, kind = 0, depth = 0;
    std::vector<int32_t> prn;
    std::vector<double> dop;
    struct Slot {
        DevBuf<float2> iq;
        DevBuf<CellRecord> rec;
        PinnedBuf<float2> h_iq;       // staging, only when the caller's IQ is pageable
        PinnedBuf<CellRecord> h_rec;  // staging, only when the caller's record buffer is pageable
        gb200_cell_record* out = nullptr;  // where this batch's records go
        bool staged_out = false;
        cudaEvent_t h2d = nullptr, done = nullptr, d2h = nullptr;
    };
    std::vector<Slot> slots;
    cudaStream_t s_in = nullptr, s_out = nullptr;
    long long head = 0, tail = 0;  // batches submitted / collected
};

// Device-resident rolling window of the newest milliseconds; every millisecond is stored at slot k and at slot
// k + capacity, so the newest n <= capacity milliseconds are contiguous whatever the write position.
struct gb200_ring {
    gb200_engine* e = nullptr;
    int capacity = 0;
    int64_t appended = 0;
    DevBuf<float2> buf;        // [2 * capacity][N]
    PinnedBuf<float2> h_stage;  // staging for pageable callers
};

namespace {

thread_local std::string g_create_error;

int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return (v && *v) ? atoi(v) : dflt;
}

// How many of a CTA's slots (correlate_slots: warps or warp pairs) share one cell.  With plenty of cells per slot each
// slot keeps a whole cell (no cross-slot merge, no CTA-wide barrier); small launches split a cell's polyphase branches
// over slots to fill the machine.
int pick_rsplit(const gb200_engine* e, int slots, long long n_cells) {
    if (n_cells >= 8LL * e->num_sms * slots) return 1;
    return std::gcd(e->s, slots);
}

size_t unit_floats2(const gb200_engine* e, int M) { return static_cast<size_t>(M) * e->s * 2 * kFft; }

// How a grid's milliseconds are integrated before their magnitudes are added: coherent segments of T milliseconds
// (T = 1: the non-coherent grid), and for a weak grid (B >= 1) B bit phases T / B milliseconds apart, each millisecond
// realigned by its code Doppler.  B = 0: the segments start at the block's first millisecond, with no realignment.
struct Segments {
    int T = 1, B = 0;
    int step() const { return B > 0 ? T / B : 0; }
    int count(int M) const { return (M - (B > 0 ? B - 1 : 0) * step()) / T; }  // K, spectra per unit
};

// doppler_spectra of n_units (block, Doppler) units, n_doppler per block, blocks of M milliseconds consecutive from iq.
// pfa: for the one-warp correlate kernel (spectra_pfa).  seg.T > 1 or a weak grid: one spectrum per segment of T
// milliseconds (seg.count(M) per unit) instead of one per millisecond; a weak grid's n_doppler folds its B bit phases.
int run_spectra(gb200_engine* e, const float2* iq, int M, const double* dop, int n_doppler, int n_units, bool pfa,
                Segments seg = {}) {
    SpectraArgs sa{};
    sa.iq = iq;
    sa.doppler = dop;
    sa.spec = e->spec.p;
    sa.tw1 = e->tw1.p;
    sa.tw2 = e->tw2.p;
    sa.block_stride = static_cast<long long>(M) * e->N;
    sa.inv_fs = 1.0 / static_cast<double>(e->fs);
    sa.N = e->N;
    sa.s = e->s;
    sa.M = seg.count(M);
    sa.T = seg.T;
    sa.align = seg.B > 0 ? 1 : 0;
    sa.phase_step = seg.step();
    sa.phase_dopplers = seg.B > 0 ? n_doppler / seg.B : 0;
    sa.n_doppler = n_doppler;
    sa.n_units = n_units;
    sa.pfa = pfa ? 1 : 0;
    GB_LAUNCH(e, 0, launch_doppler_spectra(sa, e->stream));
    return GB200_OK;
}

// The correlate arguments every launch sets; the caller adds its grid- or list-mode plan.
CorrelateArgs correlate_args(const gb200_engine* e, int M, int kind, int rsplit, CellRecord* records, float* profile) {
    CorrelateArgs ca{};
    ca.spec = e->spec.p;
    ca.crep = e->crep.p;
    ca.crep1023 = e->crep1023.p;
    ca.tw1 = e->tw1.p;
    ca.tw2 = e->tw2.p;
    ca.records = records;
    ca.profile = profile;
    ca.N = e->N;
    ca.s = e->s;
    ca.M = M;
    ca.kind = kind;
    ca.rsplit = rsplit;
    return ca;
}

// One fused block-per-cell launch (a CTA per cell, the whole pipeline in one kernel; configured on first use) over n_cells
// cells, each with its Doppler, replica row and optional coherent probe index (probe may be null).
int launch_fused(gb200_engine* e, int M, int kind, const double* doppler, const int* prn, const int* probe, CellRecord* records,
                 int n_cells) {
    if (!e->fused_configured) {
        GB_CUDA(e, configure_fused_kernel());
        e->fused_configured = true;
    }
    FusedArgs fa{};
    fa.iq = e->iq;
    fa.crep = e->crep.p;
    fa.tw1 = e->tw1.p;
    fa.tw2 = e->tw2.p;
    fa.inv_fs = 1.0 / static_cast<double>(e->fs);
    fa.N = e->N;
    fa.M = M;
    fa.doppler = doppler;
    fa.prn = prn;
    fa.probe = probe;
    fa.records = records;
    fa.n_cells = n_cells;
    GB_LAUNCH(e, 1, launch_acquire_fused(fa, e->s, kind, e->stream));
    return GB200_OK;
}

// A list-mode correlate plan: cells sorted by PRN (cell_u: spectrum unit, cell_out: record slot) and groups of consecutive
// cells of one PRN.  It lives in an int buffer as [cell_u][cell_out][grp_first][grp_count][grp_prn].
struct ListPlan {
    std::vector<int> cell_u, cell_out, grp_first, grp_count, grp_prn;
    size_t size() const { return 2 * cell_u.size() + 3 * grp_prn.size(); }
    void write(int* host) const {
        for (const auto* v : {&cell_u, &cell_out, &grp_first, &grp_count, &grp_prn}) host = std::copy(v->begin(), v->end(), host);
    }
    // Points ca at n_groups groups from group g0 on of the plan written at dev.
    void bind(CorrelateArgs& ca, const int* dev, int g0, int n_groups) const {
        const size_t nc = cell_u.size(), ng = grp_prn.size();
        ca.n_groups = n_groups;
        ca.cell_u = dev;
        ca.cell_out = dev + nc;
        ca.grp_first = dev + 2 * nc + g0;
        ca.grp_count = dev + 2 * nc + ng + g0;
        ca.grp_prn = dev + 2 * nc + 2 * ng + g0;
    }
};

// The split pipeline over groups [g0, g0 + n_groups) of the plan written at dev: doppler_spectra of the n_units Dopplers at
// dop (spectrum unit u holds dop[u]), then correlate_cells.  probe, gate and profile are optional (see CorrelateArgs).
int run_list(gb200_engine* e, const ListPlan& plan, const int* dev, int g0, int n_groups, int M, int kind, int rsplit,
             const double* dop, int n_units, CellRecord* records, const int* probe, const double* gate, float* profile) {
    GB_TRY(run_spectra(e, e->iq, M, dop, n_units, n_units, spectra_pfa(kind, profile != nullptr)));
    CorrelateArgs ca = correlate_args(e, M, kind, rsplit, records, profile);
    plan.bind(ca, dev, g0, n_groups);
    ca.cell_probe = probe;
    ca.cell_gate = gate;
    GB_LAUNCH(e, 1, launch_correlate(ca, std::min(n_groups, e->num_sms), e->stream));
    return GB200_OK;
}

// Argument rules of the acquisition entry points, one function each (host.cuh has the ones the trackers share).
int check_kind(gb200_engine* e, int kind) {
    if (kind != GB200_COHERENT && kind != GB200_NON_COHERENT) GB_FAIL(e, GB200_EINVAL, "Unexpected integration type");
    return GB200_OK;
}

// Every Doppler a caller passes is finite.  NaN is gb200_detect's own "slot switched off" mark (k_doppler_spectra and
// k_acquire_fused skip such a bin, leaving its spectra or record unwritten), and +-inf gives a NaN carrier; the reference
// returns an all-NaN profile for both, which no record can stand for.
int check_dopplers(gb200_engine* e, const double* dop, int n) {
    for (int i = 0; i < n; ++i)
        if (!std::isfinite(dop[i])) GB_FAIL(e, GB200_EINVAL, "Doppler %d is not finite (%g Hz)", i, dop[i]);
    return GB200_OK;
}

int check_grid(gb200_engine* e, int n_blocks, int P, int D, const int32_t* prn_idx, const double* dop) {
    if (n_blocks < 1 || P < 1 || D < 1 || !prn_idx || !dop) GB_FAIL(e, GB200_EINVAL, "empty grid");
    return check_dopplers(e, dop, D);
}

// A semi-coherent grid sums coherent_ms milliseconds at a time, and every block is a whole number of such segments.
int check_segments(gb200_engine* e, int ms_per_block, int coherent_ms) {
    if (coherent_ms < 1) GB_FAIL(e, GB200_EINVAL, "coherent_ms must be at least 1 (got %d)", coherent_ms);
    if (ms_per_block % coherent_ms != 0)
        GB_FAIL(e, GB200_EINVAL, "ms_per_block (%d) is not a whole number of %d-ms coherent segments", ms_per_block, coherent_ms);
    return GB200_OK;
}

// A weak grid: B bit phases T / B milliseconds apart, each summing the same K >= 1 whole segments of T milliseconds inside
// the block, and B * D folded Doppler slots that fit an int.
int check_weak(gb200_engine* e, int ms_per_block, int coherent_ms, int bit_phases, int D) {
    if (coherent_ms < 1) GB_FAIL(e, GB200_EINVAL, "coherent_ms must be at least 1 (got %d)", coherent_ms);
    if (bit_phases < 1 || coherent_ms % bit_phases != 0)
        GB_FAIL(e, GB200_EINVAL, "bit_phases (%d) must be at least 1 and divide coherent_ms (%d)", bit_phases, coherent_ms);
    const long long span = static_cast<long long>(bit_phases - 1) * (coherent_ms / bit_phases);  // last phase's offset
    if (ms_per_block < coherent_ms + span || (ms_per_block - span) % coherent_ms != 0)
        GB_FAIL(e, GB200_EINVAL, "ms_per_block (%d) is not %lld ms plus a whole number (>= 1) of %d-ms coherent segments",
                ms_per_block, span, coherent_ms);
    if (static_cast<long long>(bit_phases) * D > INT32_MAX) GB_FAIL(e, GB200_EINVAL, "bit_phases * n_doppler exceeds an int");
    return GB200_OK;
}

// What every acquisition needs before its own arguments are looked at.
int check_common(gb200_engine* e, int n_ms, int kind) {
    GB_TRY(check_kind(e, kind));
    GB_TRY(check_replicas(e));
    return check_iq(e, n_ms);
}

// Points the engine's IQ at the n samples at buf.
void bind_iq(gb200_engine* e, const float2* buf, int64_t n) {
    e->iq = buf;
    e->iq_samples = n;
}

// Forgets the engine's IQ binding when it points into the n samples at buf, which are about to be freed.
void unbind_iq(gb200_engine* e, const float2* buf, size_t n) {
    if (e->iq >= buf && e->iq < buf + n) bind_iq(e, nullptr, 0);
}

// The grid's axes (PRN rows in d_ints, Doppler bins in d_doppler) are uploaded only when they changed -- or when a list-mode
// call (gb200_acquire_cells / gb200_detect) has reused those device buffers since.
int upload_grid_axes(gb200_engine* e, const int32_t* prn_idx, int P, const double* dop, int D) {
    auto& c = e->grid_axes;
    const bool same = c.valid && static_cast<int>(c.dop.size()) == D && static_cast<int>(c.prn.size()) == P &&
                      memcmp(c.dop.data(), dop, sizeof(double) * D) == 0 && memcmp(c.prn.data(), prn_idx, sizeof(int) * P) == 0;
    if (same) return GB200_OK;
    GB_CUDA(e, cudaStreamSynchronize(e->stream));  // staging buffers may still be in flight
    GB_CUDA(e, e->d_doppler.ensure(D));
    GB_CUDA(e, e->d_ints.ensure(P));
    GB_TRY(upload(e, e->d_doppler.p, dop, D, e->h_doubles));
    GB_TRY(upload(e, e->d_ints.p, prn_idx, P, e->h_ints));
    c.dop.assign(dop, dop + D);
    c.prn.assign(prn_idx, prn_idx + P);
    c.valid = true;
    return GB200_OK;
}

// One grid call: n_blocks blocks of M milliseconds x P PRN rows x D Dopplers, each block's milliseconds summed as seg says.
// weak: seg.B is the caller's bit_phases, held to check_weak (B = 0 included).  A weak grid has bins() = B * D folded bins,
// and run_grid reads dop as that folded list.
struct GridCall {
    int n_blocks, M;
    const int32_t* prn;
    int P;
    const double* dop;
    int D, kind;
    Segments seg;
    bool weak;
    int bins() const { return D * std::max(seg.B, 1); }
    size_t rows() const { return static_cast<size_t>(n_blocks) * P; }  // (block, PRN) rows
};

// grid mode: all cells of g, records written to rec_dev (device).  The caller has applied check_grid and the segment rule
// (check_segments or check_weak).  seg.T > 1 or a weak grid: the correlate launch is the non-coherent one over the
// seg.count(M) segment spectra of each (block, bin) unit.
int run_grid(gb200_engine* e, const GridCall& g, CellRecord* rec_dev) {
    const int n_blocks = g.n_blocks, M = g.M, P = g.P, D = g.bins(), kind = g.kind;  // D: the (folded) bins
    GB_TRY(check_common(e, M, kind));
    if (static_cast<int64_t>(n_blocks) * M * e->N > e->iq_samples)
        GB_FAIL(e, GB200_EINVAL, "grid needs %lld samples, %lld loaded", static_cast<long long>(n_blocks) * M * e->N,
                static_cast<long long>(e->iq_samples));
    GB_TRY(check_prns(e, g.prn, P));
    GB_TRY(upload_grid_axes(e, g.prn, P, g.dop, D));

    const int K = g.seg.count(M);  // spectra per unit
    const size_t unit = unit_floats2(e, K);
    const size_t per_block = unit * D;
    int nb = static_cast<int>(std::max<size_t>(1, e->spec_budget_bytes / (per_block * sizeof(float2))));
    nb = std::min(nb, n_blocks);
    GB_CUDA(e, e->spec.ensure(per_block * nb));

    const int slots = correlate_slots(kind, K, false);
    const int rsplit = pick_rsplit(e, slots, static_cast<long long>(nb) * P * D);
    const int cpg = slots / rsplit;
    for (int b0 = 0; b0 < n_blocks; b0 += nb) {
        const int nbb = std::min(nb, n_blocks - b0);
        const int chunks = (nbb * D + cpg - 1) / cpg;  // groups per PRN: its nbb*D cells in chunks of cpg
        GB_TRY(run_spectra(e, e->iq + static_cast<size_t>(b0) * M * e->N, M, e->d_doppler.p, D, nbb * D, spectra_pfa(kind, false),
                           g.seg));

        CorrelateArgs ca = correlate_args(e, K, kind, rsplit, rec_dev + static_cast<size_t>(b0) * P * D, nullptr);
        ca.n_groups = P * chunks;
        ca.grid_mode = 1;
        ca.P = P;
        ca.D = D;
        ca.n_blocks = nbb;
        ca.chunks = chunks;
        ca.prn_idx = e->d_ints.p;
        const int grid = std::min(ca.n_groups, e->num_sms);
        // L2 windows of the one-warp kernel (see the kernel; the pair kernel walks the batch as one window): a batch whose
        // spectra exceed L2 is walked in equal runs of units of about l2_window_bytes (0 = off), as long as a window still
        // gives every CTA at least l2_window_min_groups groups (the kernel's round-robin of the extra groups keeps the CTAs
        // together).
        const size_t win_bytes = e->l2_window_bytes;
        const size_t batch_bytes = static_cast<size_t>(nbb) * per_block * sizeof(float2);
        if (win_bytes && batch_bytes > win_bytes + win_bytes / 2) {
            const long long n_win = static_cast<long long>((batch_bytes + win_bytes - 1) / win_bytes);
            long long wc = (chunks + n_win - 1) / n_win;
            // a window whose P * wc groups divide evenly among the CTAs, when one exists within a quarter of the target size
            const long long q = grid / std::gcd(P, grid);
            const long long even = ((wc + q / 2) / q) * q;
            if (even > 0 && even * 4 >= wc * 3 && even * 4 <= wc * 5) wc = even;
            if (wc * P >= static_cast<long long>(e->l2_window_min_groups) * grid && wc < chunks)
                ca.win_chunks = static_cast<int>(wc);
        }
        GB_LAUNCH(e, 1, launch_correlate(ca, grid, e->stream));
    }
    return GB200_OK;
}

// list mode.  Cells are sorted by PRN and cut into chunks whose spectra fit the scratch budget.
int run_cells(gb200_engine* e, int n_cells, const int32_t* prn_idx, const double* dop, const int32_t* probe, int M,
              int kind, CellRecord* rec_dev, float* profile_dev) {
    GB_TRY(check_common(e, M, kind));
    if (n_cells < 1 || !prn_idx || !dop) GB_FAIL(e, GB200_EINVAL, "empty cell list");
    GB_TRY(check_dopplers(e, dop, n_cells));
    GB_TRY(check_samples(e, M));
    GB_TRY(check_prns(e, prn_idx, n_cells));
    e->grid_axes.valid = false;  // d_ints / d_doppler are about to be overwritten

    bool use_fused = e->fused == 1;
    if (e->fused < 0 && fused_supports(e->s) && !profile_dev) {
        // Automatic choice.  The split kernels pay off when many cells share a Doppler bin (the PRN-independent half is
        // computed once per bin); lists with mostly distinct Dopplers (the refinement passes of acquisition.py:81-101)
        // and small lists are faster through the fused block-per-cell kernel.
        std::vector<double> u(dop, dop + n_cells);
        std::sort(u.begin(), u.end());
        const long long n_unique = std::unique(u.begin(), u.end()) - u.begin();
        use_fused = n_unique * 4 > n_cells || static_cast<long long>(n_cells) * M <= 8192;
    }
    if (use_fused && fused_supports(e->s) && !profile_dev) {
        GB_CUDA(e, cudaStreamSynchronize(e->stream));
        GB_CUDA(e, e->d_ints.ensure(static_cast<size_t>(n_cells) * 2));
        GB_CUDA(e, e->h_ints.ensure(static_cast<size_t>(n_cells) * 2));
        GB_CUDA(e, e->d_doppler.ensure(n_cells));
        for (int i = 0; i < n_cells; ++i) {
            e->h_ints.p[i] = prn_idx[i];
            e->h_ints.p[n_cells + i] = probe ? probe[i] : -1;
        }
        GB_CUDA(e, cudaMemcpyAsync(e->d_ints.p, e->h_ints.p, sizeof(int) * 2 * n_cells, cudaMemcpyHostToDevice, e->stream));
        GB_TRY(upload(e, e->d_doppler.p, dop, n_cells, e->h_doubles));
        return launch_fused(e, M, kind, e->d_doppler.p, e->d_ints.p, e->d_ints.p + n_cells, rec_dev, n_cells);
    }

    const int slots = correlate_slots(kind, M, profile_dev != nullptr);
    const int rsplit = pick_rsplit(e, slots, n_cells);
    const int cpg = slots / rsplit;
    std::vector<int> order(n_cells);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return prn_idx[a] < prn_idx[b]; });

    const size_t unit = unit_floats2(e, M);
    const int max_cells = static_cast<int>(std::max<size_t>(cpg, e->spec_budget_bytes / (unit * sizeof(float2)) / cpg * cpg));

    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    // probe indices live at the front of the int buffer for the whole call, each chunk's plan behind them
    const size_t ints_needed = static_cast<size_t>(n_cells) * 3 + 3 * (static_cast<size_t>(n_cells) + 1);
    GB_CUDA(e, e->d_ints.ensure(ints_needed));
    GB_CUDA(e, e->h_ints.ensure(ints_needed));
    GB_CUDA(e, e->d_doppler.ensure(n_cells));
    for (int i = 0; i < n_cells; ++i) e->h_ints.p[i] = probe ? probe[i] : -1;
    GB_CUDA(e, cudaMemcpyAsync(e->d_ints.p, e->h_ints.p, sizeof(int) * n_cells, cudaMemcpyHostToDevice, e->stream));
    GB_CUDA(e, e->spec.ensure(unit * std::min(max_cells, n_cells)));

    int c0 = 0;
    while (c0 < n_cells) {
        // take up to max_cells sorted cells, ending on a PRN-group boundary where possible
        int c1 = std::min(n_cells, c0 + max_cells);
        // plan arrays for this chunk (indices into the chunk)
        std::map<double, int> uniq;
        std::vector<double> udop;
        ListPlan plan;
        for (int c = c0; c < c1; ++c) {
            const int orig = order[c];
            auto it = uniq.find(dop[orig]);
            int u;
            if (it == uniq.end()) {
                u = static_cast<int>(udop.size());
                uniq.emplace(dop[orig], u);
                udop.push_back(dop[orig]);
            } else {
                u = it->second;
            }
            plan.cell_u.push_back(u);
            plan.cell_out.push_back(orig);
            if (plan.grp_prn.empty() || plan.grp_prn.back() != prn_idx[orig] || plan.grp_count.back() == cpg) {
                plan.grp_first.push_back(c - c0);
                plan.grp_count.push_back(1);
                plan.grp_prn.push_back(prn_idx[orig]);
            } else {
                plan.grp_count.back()++;
            }
        }
        // the staging buffers are reused per chunk: wait for the previous chunk's copies
        if (c0 > 0) GB_CUDA(e, cudaStreamSynchronize(e->stream));
        int* di = e->d_ints.p + n_cells;
        plan.write(e->h_ints.p + n_cells);
        GB_CUDA(e, cudaMemcpyAsync(di, e->h_ints.p + n_cells, sizeof(int) * plan.size(), cudaMemcpyHostToDevice, e->stream));
        GB_TRY(upload(e, e->d_doppler.p, udop.data(), udop.size(), e->h_doubles));
        GB_TRY(run_list(e, plan, di, 0, static_cast<int>(plan.grp_prn.size()), M, kind, rsplit, e->d_doppler.p,
                        static_cast<int>(udop.size()), rec_dev, e->d_ints.p, nullptr, profile_dev));
        c0 = c1;
    }
    return GB200_OK;
}

// Where a grid call's output goes: its records, or each (block, PRN) row's best bin (acquisition.py:179-189 on the
// device), into the caller's device buffer or to the host.
enum class GridOut { records_device, records_host, best_device, best_host };

// Every gb200_acquire_grid* entry point but gb200_acquire_grid_host: the argument rules in the header's order (nothing is
// launched on an error), the grid, then its output.
int acquire_grid(gb200_engine* e, GridCall g, GridOut to, void* out) {
    if (!e) return GB200_EINVAL;
    if (!out) GB_FAIL(e, GB200_EINVAL, "null output");
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_TRY(check_grid(e, g.n_blocks, g.P, g.D, g.prn, g.dop));
    GB_TRY(g.weak ? check_weak(e, g.M, g.seg.T, g.seg.B, g.D) : check_segments(e, g.M, g.seg.T));
    std::vector<double> folded;  // a weak grid's Doppler axis: bin j * D + d holds dop[d]
    if (g.weak) {
        for (int j = 0; j < g.seg.B; ++j) folded.insert(folded.end(), g.dop, g.dop + g.D);
        g.dop = folded.data();
    }
    if (to == GridOut::records_device) return run_grid(e, g, static_cast<CellRecord*>(out));
    const size_t n_rec = g.rows() * g.bins();
    GB_CUDA(e, e->d_records.ensure(n_rec));
    BestRecord* best = static_cast<BestRecord*>(out);
    if (to == GridOut::best_host) {
        GB_CUDA(e, e->d_best.ensure(g.rows()));
        best = e->d_best.p;
    }
    GB_TRY(run_grid(e, g, e->d_records.p));
    if (to == GridOut::records_host) return download(e, static_cast<CellRecord*>(out), e->d_records.p, n_rec, e->h_records);
    GB_LAUNCH(e, -1, launch_best_bins(static_cast<int>(g.rows()), g.bins(), e->N, e->d_records.p, e->d_doppler.p, best,
                                      e->stream));
    if (to == GridOut::best_device) return GB200_OK;
    return download(e, static_cast<BestRecord*>(out), best, g.rows(), e->h_best);
}

}  // namespace

extern "C" {

int gb200_abi_version(void) { return GB200_ABI_VERSION; }

const char* gb200_last_error(const gb200_engine* e) { return e ? e->err.c_str() : g_create_error.c_str(); }

int gb200_create(int device, int fs, int n, gb200_engine** out) {
    if (!out) return GB200_EINVAL;
    *out = nullptr;
    if (n <= 0 || n % kChips != 0 || fs <= 0) {
        g_create_error = "samples_per_ms must be a positive multiple of 1023 and samples_per_second positive";
        return GB200_EINVAL;
    }
    int count = 0;
    cudaError_t ce = cudaGetDeviceCount(&count);
    if (ce != cudaSuccess || device < 0 || device >= count) {
        cudaGetLastError();
        g_create_error = std::string("no usable CUDA device (there is no CPU fallback): ") +
                         (ce != cudaSuccess ? cudaGetErrorString(ce) : "ordinal out of range");
        return GB200_ECUDA;
    }
    gb200_engine* e = new gb200_engine;
    e->device = device;
    e->fs = fs;
    e->N = n;
    e->s = n / kChips;
    // Spectra scratch per launch pair.  It does not have to stay in L2 (a launch writes and re-reads 21 MB per 16.368 Msps
    // block), and launches that carry more cells run the correlate kernel without cross-warp merges and with a shorter tail.
    e->spec_budget_bytes = static_cast<size_t>(env_int("GB200_SPEC_BUDGET_MB", 512)) << 20;
    // L2 window of the one-warp correlate kernel: 16 MB is the fastest size for the benchmark's config-2 call and for config 3
    // on the H100's 50 MB L2 (DESIGN.md §4, L2 windows).
    e->l2_window_bytes = static_cast<size_t>(std::max(0, env_int("GB200_L2_WINDOW_MB", 16))) << 20;
    e->l2_window_min_groups = env_int("GB200_L2_WINDOW_MIN_GROUPS", 2);
    auto fail = [&](cudaError_t c, const char* what) {
        g_create_error = std::string(what) + ": " + cudaGetErrorString(c);
        cudaGetLastError();
        delete e;
        return GB200_ECUDA;
    };
    if ((ce = cudaSetDevice(device)) != cudaSuccess) return fail(ce, "cudaSetDevice");
    cudaDeviceProp prop;
    if ((ce = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return fail(ce, "cudaGetDeviceProperties");
    if (prop.major != 9 || prop.minor != 0) {
        g_create_error = "this build targets sm_90a (H100) only";
        delete e;
        return GB200_ECUDA;
    }
    e->num_sms = prop.multiProcessorCount;
    if (!spectra_supports(e->s)) {
#define GB_RATE_TEXT(S) "," #S
        g_create_error = std::string("samples_per_ms / 1023 must be one of ") + (GB_FOR_EACH_RATE(GB_RATE_TEXT) + 1);  // "1,2,..."
#undef GB_RATE_TEXT
        delete e;
        return GB200_EINVAL;
    }
    if ((ce = cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking)) != cudaSuccess) return fail(ce, "cudaStreamCreate");
    e->stream = e->own_stream;
    if ((ce = configure_kernels()) != cudaSuccess) return fail(ce, "cudaFuncSetAttribute");
    if ((ce = e->tw1.ensure(kFft)) != cudaSuccess) return fail(ce, "cudaMalloc");
    if ((ce = e->tw2.ensure(kFft)) != cudaSuccess) return fail(ce, "cudaMalloc");
    if ((ce = launch_init_tables(e->tw1.p, e->tw2.p, e->stream)) != cudaSuccess) return fail(ce, "init_tables");
    e->launches++;
    if ((ce = cudaStreamSynchronize(e->stream)) != cudaSuccess) return fail(ce, "init_tables sync");
    *out = e;
    return GB200_OK;
}

int gb200_destroy(gb200_engine* e) {
    if (!e) return GB200_OK;
    cudaSetDevice(e->device);
    cudaStreamSynchronize(e->stream);
    delete e;  // ~gb200_engine releases every device / pinned allocation, the events and the stream
    return GB200_OK;
}

int gb200_set_stream(gb200_engine* e, void* st) {
    if (!e) return GB200_EINVAL;
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    e->stream = st ? static_cast<cudaStream_t>(st) : e->own_stream;
    return GB200_OK;
}

int gb200_set_replicas(gb200_engine* e, const uint8_t* chips, int n_prn) {
    if (!e) return GB200_EINVAL;
    if (!chips || n_prn < 1) GB_FAIL(e, GB200_EINVAL, "need at least one PRN code");
    for (int i = 0; i < n_prn * kChips; ++i)
        if (chips[i] > 1) GB_FAIL(e, GB200_EINVAL, "chips must be 0 or 1");
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    GB_CUDA(e, e->chips.ensure(static_cast<size_t>(n_prn) * kChips));
    GB_CUDA(e, e->crep.ensure(static_cast<size_t>(n_prn) * 2 * kFft));
    GB_CUDA(e, e->crep1023.ensure(static_cast<size_t>(n_prn) * kPfaVecF2));
    GB_CUDA(e, cudaMemcpyAsync(e->chips.p, chips, static_cast<size_t>(n_prn) * kChips, cudaMemcpyHostToDevice, e->stream));
    GB_LAUNCH(e, -1, launch_replica_spectra(e->chips.p, n_prn, e->crep.p, e->crep1023.p, e->stream));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    e->n_prn = n_prn;
    return GB200_OK;
}

int gb200_upload_iq(gb200_engine* e, const float* iq_host, int64_t n_samples) {
    if (!e) return GB200_EINVAL;
    if (!iq_host || n_samples < 0) GB_FAIL(e, GB200_EINVAL, "bad IQ buffer");
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, e->iq_own.ensure(static_cast<size_t>(std::max<int64_t>(n_samples, 1))));
    const float2* src = reinterpret_cast<const float2*>(iq_host);
    if (!is_pinned(iq_host)) {
        GB_CUDA(e, cudaStreamSynchronize(e->stream));  // staging buffer may still be in flight
        GB_CUDA(e, stage_in(e->h_iq, src, static_cast<size_t>(n_samples)));
    }
    GB_CUDA(e, cudaMemcpyAsync(e->iq_own.p, src, static_cast<size_t>(n_samples) * sizeof(float2), cudaMemcpyHostToDevice,
                               e->stream));
    bind_iq(e, e->iq_own.p, n_samples);
    return GB200_OK;
}

int gb200_bind_iq_device(gb200_engine* e, const void* iq_device, int64_t n_samples) {
    if (!e) return GB200_EINVAL;
    if (!iq_device || n_samples < 0) GB_FAIL(e, GB200_EINVAL, "bad IQ buffer");
    // the fused acquisition kernel stages the IQ with cp.async.bulk and the tracking kernel with 16-byte cp.async
    if (reinterpret_cast<uintptr_t>(iq_device) % 16 != 0) GB_FAIL(e, GB200_EINVAL, "IQ buffer must be 16-byte aligned");
    bind_iq(e, static_cast<const float2*>(iq_device), n_samples);
    return GB200_OK;
}

int gb200_acquire_grid_device(gb200_engine* e, int n_blocks, int M, const int32_t* prn_idx, int P, const double* dop, int D,
                              int kind, void* out_device) {
    return acquire_grid(e, {n_blocks, M, prn_idx, P, dop, D, kind}, GridOut::records_device, out_device);
}

int gb200_acquire_grid(gb200_engine* e, int n_blocks, int M, const int32_t* prn_idx, int P, const double* dop, int D,
                       int kind, gb200_cell_record* out_host) {
    return acquire_grid(e, {n_blocks, M, prn_idx, P, dop, D, kind}, GridOut::records_host, out_host);
}

int gb200_acquire_grid_best_device(gb200_engine* e, int n_blocks, int M, const int32_t* prn_idx, int P, const double* dop, int D,
                                   int kind, void* out_device) {
    return acquire_grid(e, {n_blocks, M, prn_idx, P, dop, D, kind}, GridOut::best_device, out_device);
}

int gb200_acquire_grid_best(gb200_engine* e, int n_blocks, int M, const int32_t* prn_idx, int P, const double* dop, int D,
                            int kind, gb200_best_record* out_host) {
    return acquire_grid(e, {n_blocks, M, prn_idx, P, dop, D, kind}, GridOut::best_host, out_host);
}

// ---------------------------------------------------------------------------------------------------------
// semi-coherent grids: the non-coherent sum of |coherent sum of coherent_ms milliseconds|.  coherent_ms == 1 is the
// non-coherent grid itself (the same kernels, launched the same way).
// ---------------------------------------------------------------------------------------------------------
int gb200_acquire_grid_semicoherent(gb200_engine* e, int n_blocks, int M, int coherent_ms, const int32_t* prn_idx, int P,
                                    const double* dop, int D, gb200_cell_record* out_host) {
    return acquire_grid(e, {n_blocks, M, prn_idx, P, dop, D, GB200_NON_COHERENT, {coherent_ms}}, GridOut::records_host, out_host);
}

int gb200_acquire_grid_semicoherent_device(gb200_engine* e, int n_blocks, int M, int coherent_ms, const int32_t* prn_idx, int P,
                                           const double* dop, int D, void* out_device) {
    return acquire_grid(e, {n_blocks, M, prn_idx, P, dop, D, GB200_NON_COHERENT, {coherent_ms}}, GridOut::records_device,
                        out_device);
}

int gb200_acquire_grid_semicoherent_best(gb200_engine* e, int n_blocks, int M, int coherent_ms, const int32_t* prn_idx, int P,
                                         const double* dop, int D, gb200_best_record* out_host) {
    return acquire_grid(e, {n_blocks, M, prn_idx, P, dop, D, GB200_NON_COHERENT, {coherent_ms}}, GridOut::best_host, out_host);
}

int gb200_acquire_grid_semicoherent_best_device(gb200_engine* e, int n_blocks, int M, int coherent_ms, const int32_t* prn_idx,
                                                int P, const double* dop, int D, void* out_device) {
    return acquire_grid(e, {n_blocks, M, prn_idx, P, dop, D, GB200_NON_COHERENT, {coherent_ms}}, GridOut::best_device, out_device);
}

// ---------------------------------------------------------------------------------------------------------
// weak grids: the semi-coherent profile at each of bit_phases segment offsets, every millisecond realigned by its code
// Doppler, over the Doppler axis folded as bit_phases * n_doppler bins (bin j * n_doppler + d: phase j, Doppler d).
// ---------------------------------------------------------------------------------------------------------
int gb200_acquire_grid_weak(gb200_engine* e, int n_blocks, int M, int coherent_ms, int bit_phases, const int32_t* prn_idx,
                            int P, const double* dop, int D, gb200_cell_record* out_host) {
    return acquire_grid(e, {n_blocks, M, prn_idx, P, dop, D, GB200_NON_COHERENT, {coherent_ms, bit_phases}, true},
                        GridOut::records_host, out_host);
}

int gb200_acquire_grid_weak_device(gb200_engine* e, int n_blocks, int M, int coherent_ms, int bit_phases, const int32_t* prn_idx,
                                   int P, const double* dop, int D, void* out_device) {
    return acquire_grid(e, {n_blocks, M, prn_idx, P, dop, D, GB200_NON_COHERENT, {coherent_ms, bit_phases}, true},
                        GridOut::records_device, out_device);
}

int gb200_acquire_grid_weak_best(gb200_engine* e, int n_blocks, int M, int coherent_ms, int bit_phases, const int32_t* prn_idx,
                                 int P, const double* dop, int D, gb200_best_record* out_host) {
    return acquire_grid(e, {n_blocks, M, prn_idx, P, dop, D, GB200_NON_COHERENT, {coherent_ms, bit_phases}, true},
                        GridOut::best_host, out_host);
}

int gb200_acquire_grid_weak_best_device(gb200_engine* e, int n_blocks, int M, int coherent_ms, int bit_phases,
                                        const int32_t* prn_idx, int P, const double* dop, int D, void* out_device) {
    return acquire_grid(e, {n_blocks, M, prn_idx, P, dop, D, GB200_NON_COHERENT, {coherent_ms, bit_phases}, true},
                        GridOut::best_device, out_device);
}

// Host to host in one call.  The first call of a shape runs eagerly (it may have to upload the axes and grow buffers,
// which synchronise); the second captures {copy-in, doppler_spectra, correlate_cells, copy-out} into a CUDA graph; from
// then on a call is: 16 KB memcpy into pinned staging, one cudaGraphLaunch, one stream synchronise, memcpy out.
int gb200_acquire_grid_host(gb200_engine* e, const float* iq_host, int n_blocks, int M, const int32_t* prn_idx, int P,
                            const double* dop, int D, int kind, gb200_cell_record* out_host) {
    if (!e) return GB200_EINVAL;
    if (!iq_host || !out_host) GB_FAIL(e, GB200_EINVAL, "null buffer");
    GB_TRY(check_grid(e, std::min(n_blocks, M), P, D, prn_idx, dop));  // blocks of no milliseconds make an empty grid too
    GB_CUDA(e, cudaSetDevice(e->device));
    const size_t n_iq = static_cast<size_t>(n_blocks) * M * e->N, n_rec = static_cast<size_t>(n_blocks) * P * D;
    const size_t spec_bytes = unit_floats2(e, M) * D * sizeof(float2) * n_blocks;
    if (e->timing || spec_bytes > e->spec_budget_bytes) {  // several scratch batches / per-kernel events: plain path
        GB_TRY(gb200_upload_iq(e, iq_host, static_cast<int64_t>(n_iq)));
        return gb200_acquire_grid(e, n_blocks, M, prn_idx, P, dop, D, kind, out_host);
    }
    GB_CUDA(e, cudaStreamSynchronize(e->stream));  // the pinned staging buffers may still be in flight
    GB_CUDA(e, e->iq_own.ensure(n_iq));
    GB_CUDA(e, e->h_iq.ensure(n_iq));
    GB_CUDA(e, e->d_records.ensure(n_rec));
    GB_CUDA(e, e->h_records.ensure(n_rec));
    // Large pinned inputs (a 10-ms window is 327 KB) are copied by the DMA engine straight from the caller's buffer: staging them
    // would cost a host memcpy.  The copy node of the graph has its source baked in, so those calls launch eagerly (a few us
    // more than a replay).  Small inputs are staged and replayed.
    const float2* h2d_src = reinterpret_cast<const float2*>(iq_host);
    const bool eager_src = n_iq * sizeof(float2) > (64u << 10) && is_pinned(iq_host);
    if (!eager_src) GB_CUDA(e, stage_in(e->h_iq, h2d_src, n_iq));
    bind_iq(e, e->iq_own.p, static_cast<int64_t>(n_iq));

    // The captured kernels read the axes from d_doppler / d_ints and the replica spectra from crep: make sure those hold THIS
    // grid's axes now (a list-mode call may have reused them since the last replay; cheap when nothing changed), and treat a
    // moved buffer (gb200_set_replicas with a larger table, a larger list-mode call) as a new shape.
    GB_TRY(check_replicas(e));
    GB_TRY(check_prns(e, prn_idx, P));
    GB_TRY(upload_grid_axes(e, prn_idx, P, dop, D));
    // Small grids: the correlate kernel stores its 32-byte records straight into pinned (device-mapped under UVA) memory --
    // posted PCIe writes at the kernel's tail instead of a separate copy node behind it -- and into the CALLER's buffer when that
    // is itself pinned, which also saves the host copy out of the staging buffer.
    const bool direct = n_rec * sizeof(CellRecord) <= (256u << 10);
    void* caller_alias = nullptr;
    const bool to_caller = direct && is_pinned(out_host, &caller_alias) && caller_alias;
    CellRecord* rec_target = to_caller ? static_cast<CellRecord*>(caller_alias) : direct ? e->h_records.p : e->d_records.p;
    auto& g = e->hg;
    auto key = [&] {
        return gb200_engine::HostGraph::Key{n_blocks, M, P, D, kind, {dop, dop + D}, {prn_idx, prn_idx + P},
                                            e->iq_own.p, e->d_records.p, e->h_iq.p, e->h_records.p, e->spec.p,
                                            e->d_doppler.p, e->d_ints.p, e->crep.p, e->crep1023.p, rec_target, e->stream};
    };
    const bool same = g.seen && g.key == key();
    auto enqueue = [&]() -> int {
        GB_CUDA(e, cudaMemcpyAsync(e->iq_own.p, h2d_src, n_iq * sizeof(float2), cudaMemcpyHostToDevice, e->stream));
        GB_TRY(run_grid(e, {n_blocks, M, prn_idx, P, dop, D, kind}, rec_target));
        if (!direct)
            GB_CUDA(e, cudaMemcpyAsync(e->h_records.p, e->d_records.p, n_rec * sizeof(CellRecord), cudaMemcpyDeviceToHost, e->stream));
        return GB200_OK;
    };
    if (eager_src) {
        GB_TRY(enqueue());
    } else if (same && g.exec) {
        GB_CUDA(e, cudaGraphLaunch(g.exec, e->stream));
        e->launches += 2;
    } else if (same && !g.exec && g.seen == 1) {
        // second call of this shape: the axes are on the device and every buffer has its size, so nothing below synchronises
        g.seen = 2;  // capture is attempted once per shape
        GB_CUDA(e, cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal));
        int rc = enqueue();
        cudaGraph_t graph = nullptr;
        cudaError_t ce = cudaStreamEndCapture(e->stream, &graph);
        if (rc == GB200_OK && ce == cudaSuccess && graph) ce = cudaGraphInstantiate(&g.exec, graph, 0);
        if (graph) cudaGraphDestroy(graph);
        if (rc != GB200_OK || ce != cudaSuccess || !g.exec) {
            cudaGetLastError();
            g.exec = nullptr;
            GB_TRY(enqueue());  // capture unavailable: stay on the eager path for this shape
        } else {
            GB_CUDA(e, cudaGraphLaunch(g.exec, e->stream));
        }
    } else {
        if (!same) {
            if (g.exec) cudaGraphExecDestroy(g.exec);
            g.exec = nullptr;
        }
        GB_TRY(enqueue());
        if (!same) {
            g.key = key();  // after the run, which may have grown the spectra scratch
            g.seen = 1;
        }
    }
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    if (!to_caller) memcpy(out_host, e->h_records.p, n_rec * sizeof(CellRecord));
    return GB200_OK;
}

// ---------------------------------------------------------------------------------------------------------
// device-resident rolling sample window (receiver.py:68,100,219)
// ---------------------------------------------------------------------------------------------------------
int gb200_ring_create(gb200_engine* e, int capacity_ms, gb200_ring** out) {
    if (!e) return GB200_EINVAL;
    if (!out) GB_FAIL(e, GB200_EINVAL, "null output");
    *out = nullptr;
    if (capacity_ms < 1) GB_FAIL(e, GB200_EINVAL, "ring capacity must be at least one millisecond");
    GB_CUDA(e, cudaSetDevice(e->device));
    gb200_ring* r = new gb200_ring;
    r->e = e;
    r->capacity = capacity_ms;
    cudaError_t ce = r->buf.ensure(static_cast<size_t>(2) * capacity_ms * e->N);
    if (ce != cudaSuccess) {
        delete r;
        cudaGetLastError();
        GB_FAIL(e, GB200_ECUDA, "ring allocation failed: %s", cudaGetErrorString(ce));
    }
    *out = r;
    return GB200_OK;
}

int gb200_ring_destroy(gb200_ring* r) {
    if (!r) return GB200_OK;
    gb200_engine* e = r->e;
    cudaSetDevice(e->device);
    cudaStreamSynchronize(e->stream);
    unbind_iq(e, r->buf.p, r->buf.cap);
    delete r;
    return GB200_OK;
}

int gb200_ring_append(gb200_ring* r, const float* iq_host, int n_ms) {
    if (!r) return GB200_EINVAL;
    gb200_engine* e = r->e;
    if (!iq_host || n_ms < 1) GB_FAIL(e, GB200_EINVAL, "need at least one whole millisecond of samples");
    if (n_ms > r->capacity) GB_FAIL(e, GB200_EINVAL, "%d ms do not fit a ring of %d ms", n_ms, r->capacity);
    GB_CUDA(e, cudaSetDevice(e->device));
    const size_t N = static_cast<size_t>(e->N);
    const float2* src = reinterpret_cast<const float2*>(iq_host);
    if (!is_pinned(iq_host)) {
        GB_CUDA(e, cudaStreamSynchronize(e->stream));  // staging buffer may still be in flight
        GB_CUDA(e, stage_in(r->h_stage, src, N * n_ms));
    }
    int done = 0;
    while (done < n_ms) {
        const int slot = static_cast<int>((r->appended + done) % r->capacity);
        const int run = std::min(n_ms - done, r->capacity - slot);
        float2* lo = r->buf.p + static_cast<size_t>(slot) * N;
        float2* hi = lo + static_cast<size_t>(r->capacity) * N;
        GB_CUDA(e, cudaMemcpyAsync(lo, src + static_cast<size_t>(done) * N, run * N * sizeof(float2), cudaMemcpyHostToDevice,
                                   e->stream));
        GB_CUDA(e, cudaMemcpyAsync(hi, lo, run * N * sizeof(float2), cudaMemcpyDeviceToDevice, e->stream));
        done += run;
    }
    r->appended += n_ms;
    return GB200_OK;
}

int gb200_ring_bind_newest(gb200_ring* r, int n_ms) {
    if (!r) return GB200_EINVAL;
    gb200_engine* e = r->e;
    if (n_ms < 1 || n_ms > r->capacity || n_ms > r->appended)
        GB_FAIL(e, GB200_EINVAL, "the ring holds %lld of at most %d ms; %d asked for",
                static_cast<long long>(std::min<int64_t>(r->appended, r->capacity)), r->capacity, n_ms);
    const int first = static_cast<int>((r->appended - n_ms) % r->capacity);
    bind_iq(e, r->buf.p + static_cast<size_t>(first) * e->N, static_cast<int64_t>(n_ms) * e->N);
    return GB200_OK;
}

int gb200_ring_appended(const gb200_ring* r, int64_t* total_ms) {
    if (!r || !total_ms) return GB200_EINVAL;
    *total_ms = r->appended;
    return GB200_OK;
}

int gb200_acquire_cells(gb200_engine* e, int n_cells, const int32_t* prn_idx, const double* dop, const int32_t* probe,
                        int n_ms, int kind, gb200_cell_record* out_host) {
    if (!e) return GB200_EINVAL;
    if (!out_host) GB_FAIL(e, GB200_EINVAL, "null output");
    GB_CUDA(e, cudaSetDevice(e->device));
    if (n_cells < 1) GB_FAIL(e, GB200_EINVAL, "empty cell list");
    GB_CUDA(e, e->d_records.ensure(n_cells));
    GB_TRY(run_cells(e, n_cells, prn_idx, dop, probe, n_ms, kind, e->d_records.p, nullptr));
    return download(e, reinterpret_cast<CellRecord*>(out_host), e->d_records.p, n_cells, e->h_records);
}

int gb200_correlation_profile(gb200_engine* e, int prn, double dop, int n_ms, int kind, float* out_host) {
    if (!e) return GB200_EINVAL;
    if (!out_host) GB_FAIL(e, GB200_EINVAL, "null output");
    GB_CUDA(e, cudaSetDevice(e->device));
    const size_t nf = static_cast<size_t>(e->N) * (kind == GB200_COHERENT ? 2 : 1);
    GB_CUDA(e, e->d_profile.ensure(nf));
    GB_CUDA(e, e->d_records.ensure(1));
    const int32_t p = prn;
    GB_TRY(run_cells(e, 1, &p, &dop, nullptr, n_ms, kind, e->d_records.p, e->d_profile.p));
    return download(e, out_host, e->d_profile.p, nf, e->h_profile);
}

int gb200_correlation_profile_replica(gb200_engine* e, const float* replica_host, double dop, int n_ms, int kind,
                                      float* out_host) {
    if (!e) return GB200_EINVAL;
    if (!replica_host || !out_host) GB_FAIL(e, GB200_EINVAL, "null buffer");
    GB_TRY(check_kind(e, kind));
    GB_TRY(check_dopplers(e, &dop, 1));
    GB_TRY(check_iq(e, n_ms));
    GB_TRY(check_samples(e, n_ms));
    GB_CUDA(e, cudaSetDevice(e->device));
    const size_t nf = static_cast<size_t>(e->N) * (kind == GB200_COHERENT ? 2 : 1);
    GB_CUDA(e, cudaStreamSynchronize(e->stream));  // staging buffers may still be in flight
    GB_CUDA(e, e->d_profile.ensure(nf));
    GB_CUDA(e, e->d_replica.ensure(e->N));
    GB_TRY(upload(e, e->d_replica.p, reinterpret_cast<const float2*>(replica_host), e->N, e->h_replica));
    GB_LAUNCH(e, -1, launch_correlate_generic(e->iq, e->d_replica.p, e->N, n_ms, dop, 1.0 / static_cast<double>(e->fs), kind,
                                              e->d_profile.p, e->stream));
    return download(e, out_host, e->d_profile.p, nf, e->h_profile);
}

int gb200_enable_kernel_timing(gb200_engine* e, int on) {
    if (!e) return GB200_EINVAL;
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    e->timing = on != 0;
    e->ev_used[0] = e->ev_used[1] = 0;
    return GB200_OK;
}

int gb200_kernel_timing(gb200_engine* e, int which, double* total_ms, int64_t* launches) {
    if (!e || which < 0 || which > 1 || !total_ms || !launches) return GB200_EINVAL;
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    double t = 0.0;
    for (size_t i = 0; i < e->ev_used[which]; ++i) {
        float ms = 0.f;
        GB_CUDA(e, cudaEventElapsedTime(&ms, e->ev[which][i].first, e->ev[which][i].second));
        t += ms;
    }
    *total_ms = t;
    *launches = static_cast<int64_t>(e->ev_used[which]);
    return GB200_OK;
}

// ---------------------------------------------------------------------------------------------------------
// on-device acquisition search (acquisition.py:70-152)
// ---------------------------------------------------------------------------------------------------------
static_assert(sizeof(gb200_acquisition_result) == sizeof(RefineResult), "ABI acquisition result must match");

int gb200_detect(gb200_engine* e, int n_sv, const int32_t* prn_idx, int n_ms, gb200_acquisition_result* out_host) {
    if (!e) return GB200_EINVAL;
    if (!out_host) GB_FAIL(e, GB200_EINVAL, "null output");
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_TRY(check_common(e, n_ms, GB200_NON_COHERENT));
    if (n_sv < 1 || !prn_idx) GB_FAIL(e, GB200_EINVAL, "no satellites to search for");
    GB_TRY(check_samples(e, n_ms));
    GB_TRY(check_prns(e, prn_idx, n_sv));

    const int MAXB = kRefineMaxBins;
    const int n_cells = n_sv * MAXB;
    const int slots = correlate_slots(GB200_NON_COHERENT, n_ms, false);
    const int rsplit = pick_rsplit(e, slots, n_cells);
    const int cpg = slots / rsplit;
    const int gps = (MAXB + cpg - 1) / cpg;  // groups per satellite
    const size_t unit = unit_floats2(e, n_ms);
    int sv_per_chunk = static_cast<int>(std::max<size_t>(1, e->spec_budget_bytes / (unit * sizeof(float2) * MAXB)));
    sv_per_chunk = std::min(sv_per_chunk, n_sv);

    // Static plans: the refinement passes (cell c = sv*MAXB + b; a chunk's spectra units restart at 0) and the coherent pass
    // (one cell per satellite), then room for the probe indices the device plans.
    ListPlan plan, coh;
    for (int sv = 0; sv < n_sv; ++sv) {
        for (int b = 0; b < MAXB; ++b) {
            plan.cell_u.push_back((sv % sv_per_chunk) * MAXB + b);
            plan.cell_out.push_back(sv * MAXB + b);
        }
        for (int g = 0; g < gps; ++g) {
            plan.grp_first.push_back(sv * MAXB + g * cpg);
            plan.grp_count.push_back(std::min(cpg, MAXB - g * cpg));
            plan.grp_prn.push_back(prn_idx[sv]);
        }
        coh.cell_u.push_back(sv);
        coh.cell_out.push_back(sv);
        coh.grp_first.push_back(sv);
        coh.grp_count.push_back(1);
        coh.grp_prn.push_back(prn_idx[sv]);
    }
    const size_t n_plans = plan.size() + coh.size();
    auto& r = e->search;
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    GB_CUDA(e, r.d_ints.ensure(n_plans + n_sv));
    GB_CUDA(e, r.h_ints.ensure(n_plans + n_sv));
    plan.write(r.h_ints.p);
    coh.write(r.h_ints.p + plan.size());
    int* di = r.d_ints.p;
    GB_CUDA(e, cudaMemcpyAsync(di, r.h_ints.p, sizeof(int) * n_plans, cudaMemcpyHostToDevice, e->stream));
    int* d_probe = di + n_plans;

    GB_CUDA(e, r.state.ensure(n_sv));
    GB_CUDA(e, r.d_doppler.ensure(static_cast<size_t>(n_cells) + n_sv));
    GB_CUDA(e, r.d_records.ensure(static_cast<size_t>(n_cells) + n_sv));
    GB_CUDA(e, r.d_results.ensure(n_sv));
    GB_CUDA(e, e->spec.ensure(unit * std::max(sv_per_chunk * MAXB, n_sv)));
    double* d_coh_doppler = r.d_doppler.p + n_cells;
    CellRecord* d_coh_records = r.d_records.p + n_cells;

    // Every (satellite, bin) cell of a refinement pass has its own Doppler, so nothing is shared between PRNs: the
    // fused block-per-cell kernel does the same arithmetic without the spectra round trip through HBM.
    const bool use_fused = fused_supports(e->s);
    if (use_fused) {
        // [n_cells] replica row of every (satellite, bin) slot, then [n_sv] one per satellite for the coherent pass
        GB_CUDA(e, r.d_cell_prn.ensure(static_cast<size_t>(n_cells) + n_sv));
        GB_CUDA(e, r.h_cell_prn.ensure(static_cast<size_t>(n_cells) + n_sv));
        for (int c = 0; c < n_cells; ++c) r.h_cell_prn.p[c] = prn_idx[c / MAXB];
        for (int sv = 0; sv < n_sv; ++sv) r.h_cell_prn.p[n_cells + sv] = prn_idx[sv];
        GB_CUDA(e, cudaMemcpyAsync(r.d_cell_prn.p, r.h_cell_prn.p, sizeof(int) * (n_cells + n_sv), cudaMemcpyHostToDevice,
                                   e->stream));
    }

    GB_LAUNCH(e, -1, launch_refine_init(n_sv, r.state.p, e->stream));
    for (double spread = 7000.0; spread >= 10.0; spread /= 2.0) {  // acquisition.py:78-89
        GB_LAUNCH(e, -1, launch_refine_plan(n_sv, spread, r.state.p, r.d_doppler.p, e->stream));
        // fused: one launch per pass, a CTA per (satellite, bin) slot, no spectra scratch
        if (use_fused)
            GB_TRY(launch_fused(e, n_ms, GB200_NON_COHERENT, r.d_doppler.p, r.d_cell_prn.p, nullptr, r.d_records.p, n_cells));
        for (int sv0 = 0; !use_fused && sv0 < n_sv; sv0 += sv_per_chunk) {
            const int nsv = std::min(sv_per_chunk, n_sv - sv0);
            GB_TRY(run_list(e, plan, di, sv0 * gps, nsv * gps, n_ms, GB200_NON_COHERENT, rsplit,
                            r.d_doppler.p + static_cast<size_t>(sv0) * MAXB, nsv * MAXB, r.d_records.p, nullptr, r.d_doppler.p,
                            nullptr));
        }
        GB_LAUNCH(e, -1, launch_refine_select(n_sv, e->N, r.d_records.p, r.d_doppler.p, r.state.p, e->stream));
    }
    // coherent integration at the kept Doppler (acquisition.py:120-136)
    GB_LAUNCH(e, -1, launch_refine_coherent_plan(n_sv, r.state.p, d_coh_doppler, d_probe, e->stream));
    if (use_fused) {
        GB_TRY(launch_fused(e, n_ms, GB200_COHERENT, d_coh_doppler, r.d_cell_prn.p + n_cells, d_probe, d_coh_records, n_sv));
    } else {
        const int crsplit = pick_rsplit(e, correlate_slots(GB200_COHERENT, n_ms, false), n_sv);
        GB_TRY(run_list(e, coh, di + plan.size(), 0, n_sv, n_ms, GB200_COHERENT, crsplit, d_coh_doppler, n_sv, d_coh_records,
                        d_probe, nullptr, nullptr));
    }
    GB_LAUNCH(e, -1, launch_refine_finalize(n_sv, r.state.p, d_coh_records, r.d_results.p, e->stream));
    return download(e, reinterpret_cast<RefineResult*>(out_host), r.d_results.p, n_sv, r.h_results);
}

// ---------------------------------------------------------------------------------------------------------
// pipelined grid batches
// ---------------------------------------------------------------------------------------------------------
int gb200_grid_stream_destroy(gb200_grid_stream* g) {
    if (!g) return GB200_OK;
    cudaSetDevice(g->e->device);
    cudaStreamSynchronize(g->e->stream);
    if (g->s_in) cudaStreamSynchronize(g->s_in);
    if (g->s_out) cudaStreamSynchronize(g->s_out);
    for (auto& sl : g->slots) {
        unbind_iq(g->e, sl.iq.p, sl.iq.cap);  // gb200_grid_stream_submit binds the slot's IQ
        if (sl.h2d) cudaEventDestroy(sl.h2d);
        if (sl.done) cudaEventDestroy(sl.done);
        if (sl.d2h) cudaEventDestroy(sl.d2h);
    }
    if (g->s_in) cudaStreamDestroy(g->s_in);
    if (g->s_out) cudaStreamDestroy(g->s_out);
    delete g;
    return GB200_OK;
}

int gb200_grid_stream_create(gb200_engine* e, int n_blocks, int M, const int32_t* prn_idx, int P, const double* dop, int D,
                             int kind, int depth, gb200_grid_stream** out) {
    if (!e) return GB200_EINVAL;
    if (!out) GB_FAIL(e, GB200_EINVAL, "null output");
    *out = nullptr;
    GB_TRY(check_grid(e, n_blocks, P, D, prn_idx, dop));
    if (depth < 1 || depth > 8) GB_FAIL(e, GB200_EINVAL, "depth must be 1..8");
    // not check_common: the stream brings its own IQ (each submit binds a slot buffer and checks it), so the engine need
    // not have any bound now -- on a fresh engine, or right after another stream took its slot buffers with it
    GB_TRY(check_kind(e, kind));
    GB_TRY(check_replicas(e));
    if (M < 1) GB_FAIL(e, GB200_EINVAL, "need at least one whole millisecond of samples");
    GB_TRY(check_prns(e, prn_idx, P));
    GB_CUDA(e, cudaSetDevice(e->device));
    gb200_grid_stream* g = new gb200_grid_stream;
    g->e = e;
    g->n_blocks = n_blocks;
    g->M = M;
    g->P = P;
    g->D = D;
    g->kind = kind;
    g->depth = depth;
    g->prn.assign(prn_idx, prn_idx + P);
    g->dop.assign(dop, dop + D);
    g->slots.resize(depth);
    const size_t n_iq = static_cast<size_t>(n_blocks) * M * e->N, n_rec = static_cast<size_t>(n_blocks) * P * D;
    cudaError_t ce = cudaStreamCreateWithFlags(&g->s_in, cudaStreamNonBlocking);
    if (ce == cudaSuccess) ce = cudaStreamCreateWithFlags(&g->s_out, cudaStreamNonBlocking);
    for (auto& sl : g->slots) {
        if (ce == cudaSuccess) ce = sl.iq.ensure(n_iq);
        if (ce == cudaSuccess) ce = sl.rec.ensure(n_rec);
        if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&sl.h2d, cudaEventDisableTiming);
        if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming);
        if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&sl.d2h, cudaEventDisableTiming);
    }
    if (ce != cudaSuccess) {
        gb200_grid_stream_destroy(g);
        cudaGetLastError();
        GB_FAIL(e, GB200_ECUDA, "grid stream allocation failed: %s", cudaGetErrorString(ce));
    }
    *out = g;
    return GB200_OK;
}

int gb200_grid_stream_submit(gb200_grid_stream* g, const float* iq_host, gb200_cell_record* out_host) {
    if (!g) return GB200_EINVAL;
    gb200_engine* e = g->e;
    if (!iq_host || !out_host) GB_FAIL(e, GB200_EINVAL, "null buffer");
    if (g->head - g->tail >= g->depth) GB_FAIL(e, GB200_ESTATE, "%d batches in flight: collect one first", g->depth);
    GB_CUDA(e, cudaSetDevice(e->device));
    auto& sl = g->slots[g->head % g->depth];
    const size_t n_iq = static_cast<size_t>(g->n_blocks) * g->M * e->N, n_rec = static_cast<size_t>(g->n_blocks) * g->P * g->D;
    // the slot's previous batch was collected, so its device buffers and staging are free
    const float2* src = reinterpret_cast<const float2*>(iq_host);
    if (!is_pinned(iq_host)) GB_CUDA(e, stage_in(sl.h_iq, src, n_iq));
    sl.out = out_host;
    sl.staged_out = !is_pinned(out_host);
    if (sl.staged_out) GB_CUDA(e, sl.h_rec.ensure(n_rec));
    GB_CUDA(e, cudaMemcpyAsync(sl.iq.p, src, n_iq * sizeof(float2), cudaMemcpyHostToDevice, g->s_in));
    GB_CUDA(e, cudaEventRecord(sl.h2d, g->s_in));
    GB_CUDA(e, cudaStreamWaitEvent(e->stream, sl.h2d, 0));
    bind_iq(e, sl.iq.p, static_cast<int64_t>(n_iq));
    GB_TRY(run_grid(e, {g->n_blocks, g->M, g->prn.data(), g->P, g->dop.data(), g->D, g->kind}, sl.rec.p));
    GB_CUDA(e, cudaEventRecord(sl.done, e->stream));
    GB_CUDA(e, cudaStreamWaitEvent(g->s_out, sl.done, 0));
    GB_CUDA(e, cudaMemcpyAsync(sl.staged_out ? reinterpret_cast<gb200_cell_record*>(sl.h_rec.p) : out_host, sl.rec.p,
                               n_rec * sizeof(CellRecord), cudaMemcpyDeviceToHost, g->s_out));
    GB_CUDA(e, cudaEventRecord(sl.d2h, g->s_out));
    g->head++;
    return GB200_OK;
}

int gb200_grid_stream_collect(gb200_grid_stream* g) {
    if (!g) return GB200_EINVAL;
    gb200_engine* e = g->e;
    if (g->head == g->tail) GB_FAIL(e, GB200_ESTATE, "no batch in flight");
    GB_CUDA(e, cudaSetDevice(e->device));
    auto& sl = g->slots[g->tail % g->depth];
    GB_CUDA(e, cudaEventSynchronize(sl.d2h));
    if (sl.staged_out)
        memcpy(sl.out, sl.h_rec.p, static_cast<size_t>(g->n_blocks) * g->P * g->D * sizeof(CellRecord));
    g->tail++;
    return GB200_OK;
}

int gb200_set_fused(gb200_engine* e, int mode) {
    if (!e) return GB200_EINVAL;
    if (mode < -1 || mode > 1) GB_FAIL(e, GB200_EINVAL, "mode must be -1 (automatic), 0 or 1");
    if (mode == 1 && !fused_supports(e->s)) GB_FAIL(e, GB200_EINVAL, "the fused kernel needs 2046 or 4092 samples per ms");
    e->fused = mode;
    return GB200_OK;
}

int gb200_launch_count(const gb200_engine* e, int64_t* out) {
    if (!e || !out) return GB200_EINVAL;
    *out = e->launches;
    return GB200_OK;
}

}  // extern "C"
