// TSV -> CSR batch loader: host parser (multi-threaded) and device parser (into a batch slot, below).
// Replaces _CsvDataset._parse_csv (reference python/lib/dataset.py:107-165; SURVEY A.0): fields split on TAB
// only, no quoting; an empty field or the NA token "-" takes its default ('' / 0 / 0.0); multi-valued
// string fields split on ',' with empty tokens dropped; strings leave the loader as Fingerprint64 values
// (the same function the GPU stage uses), so no string ever crosses PCIe.  Rows are parsed in contiguous blocks, one block per
// thread, without per-row heap allocations; keys are assembled with a parallel copy.
#include <stdlib.h>
#include <string.h>

#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "common.cuh"
#include "farmhash.cuh"
#include "tsv_rules.cuh"

namespace {
struct LineRef { const char* p; int len; };

// Persistent worker threads for the per-batch parse.  Spawning threads per call looked free (~20 us each) but a freshly created
// thread starts on its creator's core and a millisecond of work is over before the scheduler spreads the threads out: measured
// here, the eight workers of a 2048-line batch ran ONE AFTER THE OTHER (same wall time as one thread).  Workers that already
// sit on their own cores are woken instead; the calling thread takes tasks too.  One dispatch at a time (callers queue up).
class WorkerPool {
    // one dispatch: its own task counter, so a worker that wakes up late (or is still leaving the previous dispatch) can only ever
    // see "no task left" of the job it holds — never a task of a newer dispatch through stale state
    struct Job {
        const std::function<void(int)>* fn;
        int n;
        std::atomic<int> next{0}, done{0};
    };

public:
    void run(int n_tasks, const std::function<void(int)>& fn) {
        if (n_tasks <= 1) { if (n_tasks == 1) fn(0); return; }
        std::lock_guard<std::mutex> serial(dispatch_);
        ensure(n_tasks - 1);
        auto job = std::make_shared<Job>();
        job->fn = &fn; job->n = n_tasks;
        {
            std::lock_guard<std::mutex> lk(m_);
            cur_ = job;
            ++gen_;
        }
        cv_work_.notify_all();
        drain(*job);
        std::unique_lock<std::mutex> lk(m_);
        cv_done_.wait(lk, [&] { return job->done.load() == job->n; });      // every task has FINISHED: fn may go out of scope
        cur_.reset();
    }

private:
    void drain(Job& j) {                             // take tasks until none is left; the last finisher wakes the dispatcher
        for (;;) {
            const int t = j.next.fetch_add(1);
            if (t >= j.n) return;
            (*j.fn)(t);
            if (j.done.fetch_add(1) + 1 == j.n) {
                std::lock_guard<std::mutex> lk(m_);  // (under the lock: the dispatcher is either before its wait or inside it)
                cv_done_.notify_all();
            }
        }
    }
    void ensure(int n) {                             // create workers: first use, or more threads asked for than exist
        while (n_workers_ < n && n_workers_ < 63) {
            std::thread([this] {
                uint64_t seen = 0;
                for (;;) {
                    std::shared_ptr<Job> job;
                    {
                        std::unique_lock<std::mutex> lk(m_);
                        cv_work_.wait(lk, [&] { return gen_ != seen; });
                        seen = gen_;
                        job = cur_;
                    }
                    if (job) drain(*job);
                }
            }).detach();                             // detached: the workers live as long as the process (no joins at exit)
            ++n_workers_;
        }
    }
    int n_workers_ = 0;
    std::mutex dispatch_, m_;
    std::condition_variable cv_work_, cv_done_;
    std::shared_ptr<Job> cur_;
    uint64_t gen_ = 0;
};
// One pool per process, leaked on purpose (workers may outlive static destructors).  A forked child gets a NEW pool: the parent's
// workers do not exist there, and its condition variables still count them as waiters.
WorkerPool& pool() {
    static std::mutex guard;
    static WorkerPool* p = nullptr;
    static pid_t owner = 0;
    std::lock_guard<std::mutex> lk(guard);
    if (!p || owner != getpid()) { p = new WorkerPool(); owner = getpid(); }
    return *p;
}

// Per-thread parse state: nothing is allocated per row.  Tokens of a row are collected in file order as (field, key) pairs and
// written field-major with a counting sort (fields may appear in any file column order).
// (one cache-line pair per thread: the vectors' end pointers are written on every token, and neighbouring ThreadOut headers in one
// line made the worker threads bounce it between their cores — eight threads parsed no faster than one)
struct alignas(128) ThreadOut {
    std::vector<uint64_t> keys;         // keys of this thread's rows, row after row, field-major inside a row
    std::vector<uint64_t> tok_key;      // scratch: tokens of the current row
    std::vector<int32_t> tok_field;
    std::vector<int32_t> pos;           // scratch: per-field write cursor
    std::string err;
};

// Integers and floats are what strtoll / strtof make of the field (the reference's decode_csv), but the common shapes are decoded
// by the exact fast paths of tsv_rules.cuh: glibc's converters cost 30-100 ns per field (locale lookup, general rounding machinery)
// and a record holds a dozen of them.  What a fast path declines goes to libc here.
inline bool parse_int_field(const char* f, int flen, long long* out) {
    if (wd::tsv_int_fast(f, flen, out)) return true;
    char buf[48];
    if (flen >= (int)sizeof(buf)) return false;
    memcpy(buf, f, flen); buf[flen] = 0;
    char* ep = nullptr;
    *out = strtoll(buf, &ep, 10);
    return *ep == 0;
}
inline bool parse_float_field(const char* f, int flen, float* out) {
    if (wd::tsv_float_fast(f, flen, out)) return true;
    char buf[64];
    if (flen >= (int)sizeof(buf)) return false;
    memcpy(buf, f, flen); buf[flen] = 0;
    char* ep = nullptr;
    *out = strtof(buf, &ep);
    return *ep == 0;
}

// one record: appends its keys to st.keys (field-major), writes counts[F], dense[Nd], label, weight
bool parse_row(const WdTsvSpec* sp, const char* p, int len, ThreadOut& st, int32_t* counts, float* dense, float* label, float* weight, char* err) {
    const int F = sp->n_cat_fields;
    st.tok_key.clear(); st.tok_field.clear();
    for (int i = 0; i < F; ++i) counts[i] = 0;
    int col = 0;
    const char* end = p + len;
    const char* f = p;
    for (int i = 0; i < sp->n_dense_fields; ++i) dense[i] = 0.f;
    float lab = 0.f;
    while (true) {
        const char* q = (const char*)memchr(f, '\t', end - f);
        const char* fe = q ? q : end;
        if (col >= sp->n_columns) { snprintf(err, 256, "Expect %d fields but have more in record", sp->n_columns); return false; }
        const int role = sp->col_role[col], tgt = sp->col_target[col];
        const int flen = (int)(fe - f);
        const bool na = wd::tsv_is_na(f, flen);
        if (role == 0) {
            lab = wd::tsv_label(f, flen, parse_int_field);
        } else if (role == 1) {
            if (!na)
                counts[tgt] += wd::tsv_tokens(f, flen, sp->multivalue, [&](const char* t, int tl) {
                    st.tok_key.push_back(wd::fingerprint64((const uint8_t*)t, tl)); st.tok_field.push_back(tgt);
                });
        } else if (role == 2) {
            long long v = 0;
            if (!na && !parse_int_field(f, flen, &v)) { snprintf(err, 256, "Field %d in record is not a valid int32: %.*s", col, flen < 40 ? flen : 40, f); return false; }
            st.tok_key.push_back((uint64_t)v); st.tok_field.push_back(tgt); counts[tgt]++;
        } else if (role == 3) {
            float v = 0.f;
            if (!na && !parse_float_field(f, flen, &v)) { snprintf(err, 256, "Field %d in record is not a valid float: %.*s", col, flen < 40 ? flen : 40, f); return false; }
            dense[tgt] = v;
        }
        ++col;
        if (!q) break;
        f = q + 1;
    }
    if (col != sp->n_columns) { snprintf(err, 256, "Expect %d fields but have %d in record", sp->n_columns, col); return false; }
    // field-major write-out (stable inside a field)
    const size_t base = st.keys.size(), nt = st.tok_key.size();
    st.keys.resize(base + nt);
    int32_t run = 0;
    for (int i = 0; i < F; ++i) { st.pos[i] = run; run += counts[i]; }
    for (size_t j = 0; j < nt; ++j) st.keys[base + st.pos[st.tok_field[j]]++] = st.tok_key[j];
    if (label) *label = lab;
    if (weight) *weight = wd::tsv_weight(sp->use_weight, sp->pos_weight, sp->neg_weight, lab);
    return true;
}
}  // namespace

namespace {
// What the last counting call (keys_out == NULL or a capacity that turned out too small) parsed on this thread: a following call for
// the SAME lines and output arrays only has to copy the keys out — the two-call protocol (size, then fill) parses once.
struct Pending {
    bool valid = false;
    const WdTsvSpec* sp = nullptr;
    const char* first = nullptr; const char* last = nullptr;
    int32_t n_lines = 0, n_threads = 0;
    const void *offsets = nullptr, *dense = nullptr, *label = nullptr, *weight = nullptr;
    int64_t nnz = 0, bytes = 0;
    uint64_t fp_first = 0, fp_last = 0;      // the pointers alone could be a recycled allocation holding other text
};

// parse `lines` (already split) into the CSR batch; see wd_tsv_parse for the contract
int64_t parse_lines(const WdTsvSpec* sp, std::vector<LineRef>& lines, int32_t n_lines, int32_t* offsets_out, uint64_t* keys_out, int64_t keys_cap,
                    float* dense_out, float* label_out, float* weight_out, int32_t n_threads, double split_ms) {
    static const bool timing = getenv("WD_TSV_TIMING") != nullptr;
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto ms = [](auto a, auto b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    // scratch kept per calling thread across calls: a batch needs tens of MB of it, and mapping / faulting / unmapping that much
    // on every call costs more than the parsing itself (and serialises the worker threads on the kernel's address-space lock)
    static thread_local std::vector<int32_t> tl_counts;
    static thread_local std::vector<float> tl_dense_tmp;
    static thread_local std::vector<ThreadOut> tl_outs;
    static thread_local std::vector<int32_t> tl_maxlen;
    static thread_local Pending tl_pending;
    // (local references: a lambda run on a worker thread would otherwise name the WORKER's thread_local instances)
    std::vector<int32_t>& counts = tl_counts;
    std::vector<float>& dense_tmp = tl_dense_tmp;
    std::vector<ThreadOut>& outs = tl_outs;
    std::vector<int32_t>& maxlen = tl_maxlen;
    Pending& pend = tl_pending;
    const int F = sp->n_cat_fields, Nd = sp->n_dense_fields;
    if (n_threads < 1) n_threads = 1;
    if (n_threads > 64) n_threads = 64;
    if (n_threads > n_lines / 256 + 1) n_threads = n_lines / 256 + 1;       // a thread is not worth less than a few hundred rows
    auto row_lo = [&](int t) { return (int)((int64_t)n_lines * t / n_threads); };
    auto run_threads = [&](const std::function<void(int)>& fn) { pool().run(n_threads, fn); };
    const char* first = n_lines > 0 ? lines[0].p : nullptr;
    const char* last = n_lines > 0 ? lines[n_lines - 1].p : nullptr;
    int64_t bytes = 0;
    for (int i = 0; i < n_lines; ++i) bytes += lines[i].len;
    const uint64_t fp_first = n_lines > 0 ? wd::fingerprint64((const uint8_t*)lines[0].p, lines[0].len) : 0;
    const uint64_t fp_last = n_lines > 0 ? wd::fingerprint64((const uint8_t*)lines[n_lines - 1].p, lines[n_lines - 1].len) : 0;
    const bool reuse = pend.valid && pend.sp == sp && pend.first == first && pend.last == last && pend.n_lines == n_lines && pend.n_threads == n_threads &&
                       pend.offsets == offsets_out && pend.dense == dense_out && pend.label == label_out && pend.weight == weight_out && dense_out &&
                       pend.bytes == bytes && pend.fp_first == fp_first && pend.fp_last == fp_last;
    pend.valid = false;
    auto t1 = now();
    if (!reuse) {
        counts.resize((size_t)n_lines * (F > 0 ? F : 1));
        dense_tmp.resize(dense_out ? 0 : (size_t)n_lines * (Nd > 0 ? Nd : 1));
        if ((int)outs.size() < n_threads) outs.resize(n_threads);
        for (auto& o : outs) { o.keys.clear(); o.err.clear(); }
        // contiguous blocks of rows per thread
        auto work = [&](int t) {
            ThreadOut& st = outs[t];
            const int lo = row_lo(t), hi = row_lo(t + 1);
            st.pos.assign(F > 0 ? F : 1, 0);
            st.tok_key.reserve(256); st.tok_field.reserve(256);
            st.keys.reserve((size_t)(hi - lo) * (F > 0 ? F : 1));
            char err[256];
            for (int i = lo; i < hi; ++i) {
                float* d = dense_out ? dense_out + (size_t)i * Nd : dense_tmp.data() + (size_t)i * Nd;
                if (!parse_row(sp, lines[i].p, lines[i].len, st, counts.data() + (size_t)i * F, d, (sp->has_label && label_out) ? label_out + i : nullptr,
                               weight_out ? weight_out + i : nullptr, err)) {
                    st.err = err;
                    return;
                }
            }
        };
        run_threads(work);
        for (auto& o : outs) if (!o.err.empty()) { wd::set_error("%s", o.err.c_str()); return WD_EINVAL; }
        // quirk Q2 (tf_compat_pad): string fields behave like dense padded tensors -> pad every row of a string
        // field to the batch max length with Fingerprint64("")
        maxlen.assign(F > 0 ? F : 1, 0);
        if (sp->tf_compat_pad)
            for (int i = 0; i < n_lines; ++i)
                for (int f = 0; f < F; ++f) maxlen[f] = std::max(maxlen[f], counts[(size_t)i * F + f]);
    }
    auto t2 = now();
    std::vector<uint8_t> is_string(F > 0 ? F : 1, 0);
    for (int c = 0; c < sp->n_columns; ++c) if (sp->col_role[c] == 1) is_string[sp->col_target[c]] = 1;
    // output offsets: one serial pass of adds; per-thread starting offsets for the parallel key copy
    std::vector<int64_t> out_start(n_threads + 1, 0);
    int64_t nnz = 0;
    {
        int t = 0;
        for (int i = 0; i < n_lines; ++i) {
            while (t < n_threads && i == row_lo(t)) out_start[t++] = nnz;
            for (int f = 0; f < F; ++f) {
                const int cnt = counts[(size_t)i * F + f];
                if (offsets_out) offsets_out[(int64_t)i * F + f] = (int32_t)nnz;
                nnz += (sp->tf_compat_pad && is_string[f]) ? maxlen[f] : cnt;
            }
        }
        while (t <= n_threads) out_start[t++] = nnz;
    }
    if (offsets_out) offsets_out[(int64_t)n_lines * F] = (int32_t)nnz;
    if (nnz > 0x7fffffffLL) { wd::set_error("wd_tsv_parse: more than 2^31 keys in one batch"); return WD_EINVAL; }
    if (!(keys_out && keys_cap > 0) || nnz > keys_cap) {
        // counting call, or the caller's buffer is too small: nothing is copied, the parsed state stays for the follow-up call
        pend.valid = true; pend.sp = sp; pend.first = first; pend.last = last; pend.n_lines = n_lines; pend.n_threads = n_threads;
        pend.offsets = offsets_out; pend.dense = dense_out; pend.label = label_out; pend.weight = weight_out; pend.nnz = nnz;
        pend.bytes = bytes; pend.fp_first = fp_first; pend.fp_last = fp_last;
        return nnz;
    }
    auto copy = [&](int t) {
        const ThreadOut& st = outs[t];
        const int lo = row_lo(t), hi = row_lo(t + 1);
        const uint64_t* k = st.keys.data();
        int64_t o = out_start[t];
        for (int i = lo; i < hi; ++i)
            for (int f = 0; f < F; ++f) {
                const int cnt = counts[(size_t)i * F + f];
                const int outc = (sp->tf_compat_pad && is_string[f]) ? maxlen[f] : cnt;
                for (int j = 0; j < cnt; ++j) keys_out[o + j] = k[j];
                for (int j = cnt; j < outc; ++j) keys_out[o + j] = wd::kFpEmpty;
                o += outc;
                k += cnt;
            }
    };
    auto t3 = now();
    run_threads(copy);
    if (timing) fprintf(stderr, "wd_tsv_parse: split %.1f ms, parse %.1f ms%s (%d threads), offsets %.1f ms, copy %.1f ms\n", split_ms, ms(t1, t2),
                        reuse ? " (reused)" : "", n_threads, ms(t2, t3), ms(t3, now()));
    return nnz;
}
thread_local std::vector<LineRef> tl_lines;
}  // namespace

extern "C" int64_t wd_tsv_parse(const WdTsvSpec* sp, const char* text, int64_t text_len, int32_t n_lines,
                                int32_t* offsets_out, uint64_t* keys_out, int64_t keys_cap,
                                float* dense_out, float* label_out, float* weight_out, int32_t n_threads) {
    if (!sp || !text || n_lines < 0) { wd::set_error("wd_tsv_parse: bad arguments"); return WD_EINVAL; }
    auto t0 = std::chrono::steady_clock::now();
    std::vector<LineRef>& lines = tl_lines;
    lines.clear();
    lines.reserve(n_lines);
    const char* p = text;
    const char* end = text + text_len;
    while (p < end && (int)lines.size() < n_lines) {
        const char* q = (const char*)memchr(p, '\n', end - p);
        const char* le = q ? q : end;
        int len = (int)(le - p);
        if (len > 0 && p[len - 1] == '\r') --len;
        lines.push_back({p, len});
        p = q ? q + 1 : end;
    }
    if ((int)lines.size() != n_lines) { wd::set_error("wd_tsv_parse: text holds %d lines, %d requested", (int)lines.size(), n_lines); return WD_EINVAL; }
    const double split_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return parse_lines(sp, lines, n_lines, offsets_out, keys_out, keys_cap, dense_out, label_out, weight_out, n_threads, split_ms);
}

// Line index of a whole file image: starts / lengths of its non-empty lines (a trailing '\r' is not part of a line), so a shuffled
// or sharded pass over the file is a permutation of indices — the text itself is never split, copied or joined again.
extern "C" int64_t wd_tsv_index_lines(const char* text, int64_t text_len, int64_t* starts_out, int32_t* lens_out, int64_t cap) {
    if (!text || text_len < 0) { wd::set_error("wd_tsv_index_lines: bad arguments"); return WD_EINVAL; }
    int64_t n = 0;
    const char* p = text;
    const char* end = text + text_len;
    while (p < end) {
        const char* q = (const char*)memchr(p, '\n', end - p);
        const char* le = q ? q : end;
        int64_t len = le - p;
        if (len > 0) {                                          // dataset.py keeps every non-empty line ("\r" alone counts as one)
            if (len > 0x7fffffffLL) { wd::set_error("wd_tsv_index_lines: line longer than 2^31 bytes"); return WD_EINVAL; }
            if (starts_out && lens_out && n < cap) {
                starts_out[n] = p - text;
                lens_out[n] = (int32_t)((p[len - 1] == '\r') ? len - 1 : len);
            }
            ++n;
        }
        p = q ? q + 1 : end;
    }
    return n;
}

// wd_tsv_parse over lines picked by index: line i of the batch = text[starts[idx[i]] .. + lens[idx[i]]) (idx NULL: i itself).
extern "C" int64_t wd_tsv_parse_lines(const WdTsvSpec* sp, const char* text, const int64_t* starts, const int32_t* lens, const int64_t* idx,
                                      int32_t n_lines, int32_t* offsets_out, uint64_t* keys_out, int64_t keys_cap,
                                      float* dense_out, float* label_out, float* weight_out, int32_t n_threads) {
    if (!sp || !text || !starts || !lens || n_lines < 0) { wd::set_error("wd_tsv_parse_lines: bad arguments"); return WD_EINVAL; }
    std::vector<LineRef>& lines = tl_lines;
    lines.resize(n_lines);
    for (int i = 0; i < n_lines; ++i) {
        const int64_t j = idx ? idx[i] : i;
        lines[i] = {text + starts[j], lens[j]};
    }
    return parse_lines(sp, lines, n_lines, offsets_out, keys_out, keys_cap, dense_out, label_out, weight_out, n_threads, 0.0);
}

// Lines picked by index, copied out of the file image into one buffer (each followed by '\n'): the text of one batch, ready for a
// single host->device copy.  out_starts[i] = start of line i in `out`, out_starts[n] = bytes of the whole batch.
extern "C" int64_t wd_tsv_gather_lines(const char* text, const int64_t* starts, const int32_t* lens, const int64_t* idx, int32_t n,
                                       char* out, int64_t out_cap, int64_t* out_starts, int32_t n_threads) {
    if (!text || !starts || !lens || !out_starts || n < 0) { wd::set_error("wd_tsv_gather_lines: bad arguments"); return WD_EINVAL; }
    int64_t total = 0;
    for (int i = 0; i < n; ++i) {
        out_starts[i] = total;
        total += (int64_t)lens[idx ? idx[i] : i] + 1;
    }
    out_starts[n] = total;
    if (!out || total > out_cap) return total;                 // sizing call, or the buffer is too small: nothing copied
    if (n_threads < 1) n_threads = 1;
    if (n_threads > 64) n_threads = 64;
    if (n_threads > n / 256 + 1) n_threads = n / 256 + 1;
    pool().run(n_threads, [&](int t) {
        const int lo = (int)((int64_t)n * t / n_threads), hi = (int)((int64_t)n * (t + 1) / n_threads);
        for (int i = lo; i < hi; ++i) {
            const int64_t j = idx ? idx[i] : i;
            memcpy(out + out_starts[i], text + starts[j], lens[j]);
            out[out_starts[i] + lens[j]] = '\n';
        }
    });
    return total;
}

// ================================================================================================== device parser
// The batch text (lines separated by one byte, normally '\n'; a trailing '\r' is not part of a line) is copied to the device and
// parsed there into a batch slot, with the field rules of tsv_rules.cuh, in three launches on the upload stream:
//   pass 1    one warp per line: TABs found with 16-byte loads and ballots, column count checked, tokens of every categorical field
//             counted, dense fields / label / weight decoded in place
//   offsets   one block: quirk Q2 padding of string fields to their batch maximum, then an exclusive scan over (row, field)
//   pass 2    one warp per line, one lane per categorical field: Fingerprint64 of string tokens, the int of int fields, padding
// A field shape outside the fast paths, a wrong column count or too many keys sets a bit of a status word; the caller then parses
// the same lines on the host, which also yields the host parser's error messages.
namespace wd {
namespace {
constexpr int kTsvWarps = 8;                     // lines per block of the per-line passes
constexpr int kTsvDecline = 1, kTsvColumns = 2, kTsvKeys = 4;

struct TsvArgs {
    const char* text;
    const int64_t* starts;                       // [n + 1]: line i = text[starts[i], starts[i + 1] - 1)
    int n, C, F, Nd;
    int multivalue, pad, has_label, want_weight, label_col;
    float pos_weight, neg_weight;
    int use_weight;
    const int32_t* cat_col;                      // [F] column of categorical field f, -1: none
    const int32_t* cat_str;                      // [F] 1: string field
    const int32_t* dense_col;                    // [Nd] column of dense field d, -1: none
    int32_t* counts;                             // [n, F] tokens per (row, field)
    int32_t* fpos;                               // [n, C + 1] start of column c in text; [C] = end of line + 1
    int32_t* fmax;                               // [F] largest count of the batch (tf_compat_pad)
    int32_t* status;
    int32_t* off;
    uint64_t* keys;
    int64_t keys_cap;
    float *dense, *label, *weight;
};

__device__ __forceinline__ unsigned tab_bits(unsigned w) {          // bit b: byte b of w is a TAB
    const unsigned m = __vcmpeq4(w, 0x09090909u);
    return ((m >> 7) & 1u) | ((m >> 14) & 2u) | ((m >> 21) & 4u) | ((m >> 28) & 8u);
}

__global__ void __launch_bounds__(kTsvWarps * 32) tsv_pass1_kernel(TsvArgs p) {
    extern __shared__ int32_t tsv_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * kTsvWarps + warp;
    if (i >= p.n) return;
    int32_t* fs = tsv_smem + warp * (p.C + 1);
    const int64_t a = p.starts[i];
    int64_t e = p.starts[i + 1] - 1;
    if (e > a && p.text[e - 1] == '\r') --e;
    if (lane == 0) fs[0] = (int32_t)a;
    int ncol = 1;
    for (int64_t c0 = a & ~(int64_t)15; c0 < e; c0 += 512) {
        const int64_t q = c0 + lane * 16;
        unsigned mask = 0;
        if (q < e) {
            const uint4 w = *reinterpret_cast<const uint4*>(p.text + q);   // (the device buffer is padded past the text)
            mask = tab_bits(w.x) | (tab_bits(w.y) << 4) | (tab_bits(w.z) << 8) | (tab_bits(w.w) << 12);
            if (q < a) mask &= 0xFFFFu << (int)(a - q);
            if (e - q < 16) mask &= (1u << (int)(e - q)) - 1u;
        }
        const int cnt = __popc(mask);
        int incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xFFFFFFFFu, incl, o);
            if (lane >= o) incl += v;
        }
        int k = ncol + incl - cnt;                               // column that starts after this lane's first TAB
        while (mask) {
            const int b = __ffs(mask) - 1;
            mask &= mask - 1;
            if (k < p.C) fs[k] = (int32_t)(q + b + 1);
            ++k;
        }
        ncol += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
    if (ncol != p.C) {
        if (lane == 0) atomicOr(p.status, kTsvColumns);
        return;
    }
    if (lane == 0) fs[p.C] = (int32_t)e + 1;
    __syncwarp();
    for (int c = lane; c <= p.C; c += 32) p.fpos[(int64_t)i * (p.C + 1) + c] = fs[c];
    bool bad = false;
    for (int d = lane; d < p.Nd; d += 32) {
        const int c = p.dense_col[d];
        float v = 0.f;
        if (c >= 0) {
            const char* f = p.text + fs[c];
            const int len = fs[c + 1] - 1 - fs[c];
            if (!tsv_is_na(f, len) && !tsv_float_fast(f, len, &v)) { bad = true; v = 0.f; }
        }
        p.dense[(int64_t)i * p.Nd + d] = v;
    }
    for (int t = lane; t < p.F; t += 32) {
        const int c = p.cat_col[t];
        int cnt = 0;
        if (c >= 0) {
            const char* f = p.text + fs[c];
            const int len = fs[c + 1] - 1 - fs[c];
            const bool na = tsv_is_na(f, len);
            if (p.cat_str[t]) {
                if (!na) cnt = tsv_tokens(f, len, p.multivalue, [](const char*, int) {});
                if (p.pad) atomicMax(p.fmax + t, cnt);
            } else {
                long long v;
                if (!na && !tsv_int_fast(f, len, &v)) bad = true;
                cnt = 1;
            }
        }
        p.counts[(int64_t)i * p.F + t] = cnt;
    }
    if (lane == 0) {
        float lab = 0.f;
        if (p.label_col >= 0) {
            const char* f = p.text + fs[p.label_col];
            lab = tsv_label(f, fs[p.label_col + 1] - 1 - fs[p.label_col], [&](const char* s, int l, long long* v) {
                if (tsv_int_fast(s, l, v)) return true;
                bad = true;                                      // strtoll might still read 1 (" 1", "+1"): the host decides
                return false;
            });
        }
        if (p.has_label) p.label[i] = lab;
        if (p.want_weight) p.weight[i] = tsv_weight(p.use_weight, p.pos_weight, p.neg_weight, lab);
    }
    if (__any_sync(0xFFFFFFFFu, bad) && lane == 0) atomicOr(p.status, kTsvDecline);
}

// one block: per-thread runs of rows, a block scan of the runs' key totals, then the offsets of every (row, field)
__global__ void __launch_bounds__(1024) tsv_offsets_kernel(TsvArgs p) {
    extern __shared__ int32_t tsv_smem[];
    __shared__ long long wsum[32];
    if (*p.status) return;
    const int F = p.F, n = p.n;
    int32_t* fixed = tsv_smem;                                   // [F] padded count of a string field, -1: the row's own count
    for (int f = threadIdx.x; f < F; f += blockDim.x) fixed[f] = (p.pad && p.cat_str[f]) ? p.fmax[f] : -1;
    __syncthreads();
    const int per = (n + blockDim.x - 1) / blockDim.x;
    const int lo = min(n, (int)threadIdx.x * per), hi = min(n, lo + per);
    long long s = 0;
    for (int i = lo; i < hi; ++i)
        for (int f = 0; f < F; ++f) s += fixed[f] >= 0 ? fixed[f] : p.counts[(int64_t)i * F + f];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    long long incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long v = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const int nw = blockDim.x >> 5;
        long long w = lane < nw ? wsum[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long v = __shfl_up_sync(0xFFFFFFFFu, w, o);
            if (lane >= o) w += v;
        }
        if (lane < nw) wsum[lane] = w;                           // inclusive over warps
    }
    __syncthreads();
    long long o = incl - s + (warp > 0 ? wsum[warp - 1] : 0);
    for (int i = lo; i < hi; ++i)
        for (int f = 0; f < F; ++f) {
            p.off[(int64_t)i * F + f] = (int32_t)o;
            o += fixed[f] >= 0 ? fixed[f] : p.counts[(int64_t)i * F + f];
        }
    if (threadIdx.x == blockDim.x - 1) {
        const long long total = wsum[(blockDim.x >> 5) - 1];
        p.off[(int64_t)n * F] = (int32_t)total;
        if (total > p.keys_cap) atomicOr(p.status, kTsvKeys);
    }
}

__global__ void __launch_bounds__(kTsvWarps * 32) tsv_pass2_kernel(TsvArgs p) {
    if (*p.status) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * kTsvWarps + warp;
    if (i >= p.n) return;
    const int32_t* fs = p.fpos + (int64_t)i * (p.C + 1);
    for (int t = lane; t < p.F; t += 32) {
        int64_t o = p.off[(int64_t)i * p.F + t];
        const int64_t oe = p.off[(int64_t)i * p.F + t + 1];
        const int c = p.cat_col[t];
        if (c >= 0) {
            const char* f = p.text + fs[c];
            const int len = fs[c + 1] - 1 - fs[c];
            const bool na = tsv_is_na(f, len);
            if (p.cat_str[t]) {
                if (!na) tsv_tokens(f, len, p.multivalue, [&](const char* s, int l) { p.keys[o++] = fingerprint64((const uint8_t*)s, l); });
            } else {
                long long v = 0;
                if (!na) tsv_int_fast(f, len, &v);
                p.keys[o++] = (uint64_t)v;
            }
        }
        for (; o < oe; ++o) p.keys[o] = kFpEmpty;
    }
}

int grow(void** ptr, int64_t* cap, int64_t need) {              // device scratch of at least `need` bytes (contents not kept)
    if (need <= *cap) return WD_OK;
    need = need + need / 4 + 256;
    if (*ptr) cudaFree(*ptr);
    *ptr = nullptr; *cap = 0;
    WD_CUDA(cudaMalloc(ptr, (size_t)need));
    *cap = need;
    return WD_OK;
}
}  // namespace

// Device state of the parser: the last spec seen (its role / target arrays, inverted into per-field columns on the device) and
// scratch of its own — a parse overlaps the step on the model stream, so it shares no buffer with it.
struct TsvDev {
    std::vector<int32_t> role, target;
    int32_t n_cat = -1, n_dense = -1;
    bool eligible = false;
    int label_col = -1;
    std::vector<int32_t> h_map;                  // [F] cat column | [F] is string | [Nd] dense column
    int32_t* d_map = nullptr; int64_t map_cap = 0;
    char* d_text = nullptr; int64_t text_cap = 0;
    int64_t* d_starts = nullptr; int64_t starts_cap = 0;
    int32_t* d_counts = nullptr; int64_t counts_cap = 0;
    int32_t* d_fpos = nullptr; int64_t fpos_cap = 0;
    int32_t* d_small = nullptr; int64_t small_cap = 0;       // [0] status, [1 .. F] fmax
    int32_t* h_status = nullptr;                 // page-locked copy of the status word
    cudaEvent_t ev = nullptr;
};

void tsv_dev_destroy(WdModel* m) {
    TsvDev* t = m->tsv;
    if (!t) return;
    for (void* p : {(void*)t->d_map, (void*)t->d_text, (void*)t->d_starts, (void*)t->d_counts, (void*)t->d_fpos, (void*)t->d_small})
        if (p) cudaFree(p);
    if (t->h_status) cudaFreeHost(t->h_status);
    if (t->ev) cudaEventDestroy(t->ev);
    delete t;
    m->tsv = nullptr;
}

// the spec's per-column arrays as per-field columns; a spec the device parser does not take (two columns feeding one field, more
// than one label column, fields other than the model's) stays on the host path
static int tsv_dev_spec(WdModel* m, TsvDev* t, const WdTsvSpec* sp, cudaStream_t st) {
    const int C = sp->n_columns;
    if (C == (int)t->role.size() && sp->n_cat_fields == t->n_cat && sp->n_dense_fields == t->n_dense &&
        (C == 0 || (!memcmp(t->role.data(), sp->col_role, C * 4) && !memcmp(t->target.data(), sp->col_target, C * 4))))
        return WD_OK;
    t->role.assign(sp->col_role, sp->col_role + C);
    t->target.assign(sp->col_target, sp->col_target + C);
    t->n_cat = sp->n_cat_fields; t->n_dense = sp->n_dense_fields;
    const int F = sp->n_cat_fields, Nd = sp->n_dense_fields;
    t->eligible = C >= 1 && F == m->n_cat_fields && Nd == m->n_dense_fields;
    t->label_col = -1;
    t->h_map.assign((size_t)2 * F + Nd, -1);
    for (int f = 0; f < F; ++f) t->h_map[F + f] = 0;
    for (int c = 0; c < C && t->eligible; ++c) {
        const int r = t->role[c], g = t->target[c];
        if (r == 0) {
            t->eligible = t->label_col < 0;
            t->label_col = c;
        } else if (r == 1 || r == 2) {
            t->eligible = g >= 0 && g < F && t->h_map[g] < 0;
            if (t->eligible) { t->h_map[g] = c; t->h_map[F + g] = r == 1; }
        } else if (r == 3) {
            t->eligible = g >= 0 && g < Nd && t->h_map[2 * F + g] < 0;
            if (t->eligible) t->h_map[2 * F + g] = c;
        } else {
            t->eligible = r == -1;
        }
    }
    if (!t->eligible) return WD_OK;
    int rc;
    if ((rc = grow((void**)&t->d_map, &t->map_cap, (int64_t)t->h_map.size() * 4 + 4))) return rc;
    WD_CUDA(cudaMemcpyAsync(t->d_map, t->h_map.data(), t->h_map.size() * 4, cudaMemcpyHostToDevice, st));
    return WD_OK;
}

// Parse n lines on stream `st` into the given batch buffers and wait for that work alone.  *status: 0 = the buffers hold the batch,
// non-zero = they do not (a decline, or a spec / batch the device parser does not take): parse on the host.
int tsv_parse_device(WdModel* m, const WdTsvSpec* sp, const char* text, int64_t text_len, const int64_t* starts, int n, int32_t* off,
                     uint64_t* keys, float* dense, float* label, float* weight, cudaStream_t st, int* status) {
    *status = -1;
    if (!m->tsv) m->tsv = new TsvDev();
    TsvDev* t = m->tsv;
    int rc;
    if ((rc = tsv_dev_spec(m, t, sp, st))) return rc;
    if (!t->eligible || n < 1 || n > m->max_batch || text_len >= 0x7fffffffLL) return WD_OK;
    const int C = sp->n_columns, F = sp->n_cat_fields, Nd = sp->n_dense_fields;
    const int64_t last = starts[n] - 1;                           // the byte after the last line
    if (starts[0] < 0 || last > text_len) return WD_OK;
    for (int i = 0; i < n; ++i) if (starts[i + 1] <= starts[i]) return WD_OK;
    if (!t->ev) WD_CUDA(cudaEventCreateWithFlags(&t->ev, cudaEventDisableTiming));
    if (!t->h_status) WD_CUDA(cudaHostAlloc((void**)&t->h_status, 64, cudaHostAllocPortable));
    if ((rc = grow((void**)&t->d_text, &t->text_cap, text_len + 64))) return rc;
    if ((rc = grow((void**)&t->d_starts, &t->starts_cap, (int64_t)(n + 1) * 8))) return rc;
    if ((rc = grow((void**)&t->d_counts, &t->counts_cap, (int64_t)n * std::max(F, 1) * 4))) return rc;
    if ((rc = grow((void**)&t->d_fpos, &t->fpos_cap, (int64_t)n * (C + 1) * 4))) return rc;
    if ((rc = grow((void**)&t->d_small, &t->small_cap, (int64_t)(F + 1) * 4))) return rc;
    WD_CUDA(cudaMemcpyAsync(t->d_text, text, text_len, cudaMemcpyHostToDevice, st));
    WD_CUDA(cudaMemcpyAsync(t->d_starts, starts, (int64_t)(n + 1) * 8, cudaMemcpyHostToDevice, st));
    WD_CUDA(cudaMemsetAsync(t->d_small, 0, (int64_t)(F + 1) * 4, st));
    TsvArgs p{};
    p.text = t->d_text; p.starts = t->d_starts; p.n = n; p.C = C; p.F = F; p.Nd = Nd;
    p.multivalue = sp->multivalue; p.pad = sp->tf_compat_pad; p.has_label = sp->has_label;
    p.use_weight = sp->use_weight; p.want_weight = sp->use_weight && sp->has_label; p.label_col = t->label_col;
    p.pos_weight = sp->pos_weight; p.neg_weight = sp->neg_weight;
    p.cat_col = t->d_map; p.cat_str = t->d_map + F; p.dense_col = t->d_map + 2 * F;
    p.counts = t->d_counts; p.fpos = t->d_fpos; p.status = t->d_small; p.fmax = t->d_small + 1;
    p.off = off; p.keys = keys; p.keys_cap = m->keys_cap; p.dense = dense; p.label = label; p.weight = weight;
    const int blocks = (n + kTsvWarps - 1) / kTsvWarps;
    tsv_pass1_kernel<<<blocks, kTsvWarps * 32, kTsvWarps * (C + 1) * 4, st>>>(p);
    tsv_offsets_kernel<<<1, 1024, std::max(F, 1) * 4, st>>>(p);
    tsv_pass2_kernel<<<blocks, kTsvWarps * 32, 0, st>>>(p);
    WD_CUDA(cudaGetLastError());
    m->launches += 3;
    WD_CUDA(cudaMemcpyAsync(t->h_status, t->d_small, 4, cudaMemcpyDeviceToHost, st));
    WD_CUDA(cudaEventRecord(t->ev, st));
    WD_CUDA(cudaEventSynchronize(t->ev));
    *status = t->h_status[0];
    return WD_OK;
}

// The same lines through the host parser, into buffers kept per calling thread: *out views them until the next call.
int tsv_parse_host(const WdTsvSpec* sp, const char* text, const int64_t* starts, int n, WdBatch* out) {
    static thread_local std::vector<LineRef> lines;
    static thread_local std::vector<int32_t> offsets;
    static thread_local std::vector<uint64_t> keys;
    static thread_local std::vector<float> dense, label, weight;
    const int F = sp->n_cat_fields, Nd = sp->n_dense_fields;
    lines.resize(n > 0 ? n : 0);
    for (int i = 0; i < n; ++i) {
        int len = (int)(starts[i + 1] - 1 - starts[i]);
        if (len > 0 && text[starts[i] + len - 1] == '\r') --len;
        lines[i] = {text + starts[i], len};
    }
    offsets.resize((size_t)std::max(n, 0) * F + 1);
    dense.resize((size_t)std::max(n, 1) * std::max(Nd, 1));
    label.resize(std::max(n, 1));
    weight.resize(std::max(n, 1));
    const int threads = (int)std::min(16u, std::max(1u, std::thread::hardware_concurrency()));
    int64_t nnz = parse_lines(sp, lines, n, offsets.data(), nullptr, 0, dense.data(), label.data(), weight.data(), threads, 0.0);
    if (nnz < 0) return (int)nnz;
    keys.resize(std::max<int64_t>(nnz, 1));
    nnz = parse_lines(sp, lines, n, offsets.data(), keys.data(), (int64_t)keys.size(), dense.data(), label.data(), weight.data(), threads, 0.0);
    if (nnz < 0) return (int)nnz;
    out->batch_size = n;
    out->cat_offsets = offsets.data();
    out->cat_keys = keys.data();
    out->nnz = nnz;
    out->dense = dense.data();
    out->label = sp->has_label ? label.data() : nullptr;
    out->weight = (sp->use_weight && sp->has_label) ? weight.data() : nullptr;
    return WD_OK;
}
}  // namespace wd

// Page-locked host memory for the input pipeline (dataset.py parses TSV text straight into a ring of these buffers, so the
// asynchronous refill of a batch slot, wd_batch_prefetch_slot, really is asynchronous).  Counterpart of the buffers tf.data's
// prefetch owns in the reference's input_fn (python/lib/dataset.py:181-184).
extern "C" int wd_host_alloc(size_t bytes, void** out) {
    if (!out) { wd::set_error("wd_host_alloc: null output"); return WD_EINVAL; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { wd::set_error("no CUDA device: cannot page-lock host memory"); return WD_ENODEVICE; }
    void* p = nullptr;
    cudaError_t e = cudaHostAlloc(&p, bytes > 0 ? bytes : 1, cudaHostAllocPortable);
    if (e != cudaSuccess) { wd::set_error("cudaHostAlloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); return WD_ENOMEM; }
    *out = p;
    return WD_OK;
}
extern "C" int wd_host_free(void* p) {
    if (p) cudaFreeHost(p);
    return WD_OK;
}
