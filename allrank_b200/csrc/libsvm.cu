// LibSVM / SVMlight text -> the SlateStore arrays, on the device (sklearn.datasets.load_svmlight_file(f,
// query_id=True) followed by SlateStore.__init__, bit for bit).  DESIGN.md section 11.
//
//   lf_count_kernel / lf_write_kernel   the line index: each block counts the '\n' of a 64 KB chunk; the counts are
//                                       scanned; each block then writes the positions of its newlines in order.
//   pass1_kernel                        one warp per line: tokens, grammar, qid, smallest / largest feature index and
//                                       a status; per-warp results folded into an 8-word summary with integer atomics
//                                       (min / max / add: the same result in any order).  The row flags are then
//                                       scanned into row numbers.
//   pass2_kernel                        one warp per row line: writes the whole dense row docs_x[r, :] (zeros first,
//                                       then the values), docs_y[r] and the row's qid; float32 as SlateStore keeps
//                                       them, or float64 as load_svmlight_file(...).toarray() returns them.
// Lines are split at '\n' only, as Python iterates over a binary file; a line is cut at its first '#' unless a NUL
// byte comes before it (sklearn's strchr stops there); tokens are
// separated by ASCII whitespace (space \t \r \v \f), as bytes.split() does.  A line with no token is not a row.
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

#include "common.h"
#include "libsvm_numeral.cuh"
#include "libsvm_scan.cuh"

namespace arb {

constexpr int LF_CHUNK = 1 << 16;       // bytes per block of the newline kernels
constexpr int LF_THREADS = 256;         // x 16 bytes = 4 KB per block step
constexpr int SVM_WARPS = 8;            // warps per block of the line kernels

// summary words (int64) of pass 1
enum { SUM_ERROR = 0, SUM_MIN_INDEX = 1, SUM_MAX_INDEX = 2, SUM_ROWS = 3, SUM_NO_QID = 4, SUM_WORDS = 8 };

__device__ __forceinline__ int nl_in_word(uint32_t w) { return __popc(__vcmpeq4(w, 0x0a0a0a0au)) >> 3; }

__device__ __forceinline__ bool svm_space(uint8_t c) {
  return c == ' ' || c == '\t' || c == '\r' || c == '\v' || c == '\f' || c == '\n';
}

// newline count of bytes [p, min(p + 16, n)) (p is 16-byte aligned relative to the 256-byte-aligned buffer)
__device__ __forceinline__ int count16(const uint8_t* text, long long p, long long n) {
  if (p + 16 <= n) {
    const uint4 v = *reinterpret_cast<const uint4*>(text + p);
    return nl_in_word(v.x) + nl_in_word(v.y) + nl_in_word(v.z) + nl_in_word(v.w);
  }
  int c = 0;
  for (long long q = p; q < n; ++q) c += text[q] == '\n';
  return c;
}

__global__ void __launch_bounds__(LF_THREADS) lf_count_kernel(const uint8_t* __restrict__ text, long long n,
                                                              long long* __restrict__ counts) {
  const long long beg = (long long)blockIdx.x * LF_CHUNK;
  const long long end = beg + LF_CHUNK < n ? beg + LF_CHUNK : n;
  int c = 0;
  for (long long p = beg + threadIdx.x * 16; p < end; p += LF_THREADS * 16) c += count16(text, p, end);
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  __shared__ int red[LF_THREADS / 32];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long t = 0;
    for (int w = 0; w < LF_THREADS / 32; ++w) t += red[w];
    counts[blockIdx.x] = t;
  }
}

// line_end[first newline of the chunk + k] = position of its k-th newline
__global__ void __launch_bounds__(LF_THREADS) lf_write_kernel(const uint8_t* __restrict__ text, long long n,
                                                              const long long* __restrict__ chunk_first,
                                                              long long* __restrict__ line_end) {
  const long long beg = (long long)blockIdx.x * LF_CHUNK;
  const long long end = beg + LF_CHUNK < n ? beg + LF_CHUNK : n;
  __shared__ int warp_tot[LF_THREADS / 32];
  long long base = chunk_first[blockIdx.x];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (long long step = beg; step < end; step += LF_THREADS * 16) {
    const long long p = step + threadIdx.x * 16;
    const int c = p < end ? count16(text, p, end) : 0;
    int incl = c;
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += v;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    int before = incl - c, total = 0;
    for (int w = 0; w < LF_THREADS / 32; ++w) {
      if (w < wid) before += warp_tot[w];
      total += warp_tot[w];
    }
    if (c) {
      long long o = base + before;
      const long long stop = p + 16 < end ? p + 16 : end;
      for (long long q = p; q < stop; ++q)
        if (text[q] == '\n') line_end[o++] = q;
    }
    base += total;
    __syncthreads();
  }
}

// What one line holds (pass 1) -- or, in pass 2, the writes it makes.
struct LineScan {
  int status;             // ARB_LIBSVM_E_* of the first failing token (0: none)
  long long ntok;
  int min_idx, max_idx;   // over the line's features (INT_MAX / -1 when it has none)
  bool has_qid;
  long long qid;
};

__device__ __forceinline__ long long token_end(const uint8_t* text, long long t, long long cut) {
  while (t < cut && !svm_space(text[t])) ++t;
  return t;
}

// What pass 2 stores for a numeral: float32 as SlateStore keeps it (sklearn_f32_bits), or float64 as
// load_svmlight_file(...).toarray() gives it -- float(token), with a feature's -0.0 added into the zeroed array (+0.0).
__device__ __forceinline__ void store_feature(float* p, double v) {
  *p = __uint_as_float(svm::sklearn_f32_bits(v, true));
}
__device__ __forceinline__ void store_feature(double* p, double v) { *p = v == 0.0 ? 0.0 : v; }
__device__ __forceinline__ void store_label(float* p, double v) {
  *p = __uint_as_float(svm::sklearn_f32_bits(v, false));
}
__device__ __forceinline__ void store_label(double* p, double v) { *p = v; }

// Walks line [beg, end) in 32-byte windows.  Token starts come from ballots over whitespace; each start lane parses
// its own token.  WRITE (pass 2): feature values go to xrow[idx - shift], the label to *y_out.
template <bool WRITE, typename T = float>
__device__ LineScan scan_line(const uint8_t* __restrict__ text, long long beg, long long end, int shift,
                              T* __restrict__ xrow, T* __restrict__ y_out) {
  const int lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1u;
  LineScan r{0, 0, 0x7fffffff, -1, false, 0};
  long long cut = end;
  unsigned carry_ws = 1;        // the byte before the window is whitespace (or the line start)
  int prev_idx = -1;            // sklearn's prev_idx: the last feature index of the line so far
  bool cuttable = true;          // sklearn cuts at strchr(line, '#'), which stops at a NUL byte
  for (long long p = beg; p < cut; p += 32) {
    const long long q = p + lane;
    uint8_t c = q < cut ? text[q] : uint8_t(' ');
    if (cuttable) {
      const unsigned hash = __ballot_sync(0xffffffffu, c == '#');
      const unsigned nul = __ballot_sync(0xffffffffu, c == 0 && q < cut);
      const int first_hash = hash ? __ffs(hash) - 1 : 32, first_nul = nul ? __ffs(nul) - 1 : 32;
      if (first_hash < first_nul) {
        cut = p + first_hash;
        if (q >= cut) c = ' ';
      } else if (nul) {
        cuttable = false;        // a NUL before any '#': the line is not cut at all
      }
    }
    const unsigned W = __ballot_sync(0xffffffffu, svm_space(c));
    const unsigned S = ~W & ((W << 1) | carry_ws);
    carry_ws = W >> 31;
    if (!S) continue;
    const bool me = (S >> lane) & 1u;
    const long long ord = r.ntok + __popc(S & lt);
    int code = 0, idx = -1;
    long long qid = 0;
    bool is_qid = false;
    if (me) {
      const long long te = token_end(text, q, cut);
      const uint8_t* tok = text + q;
      const long long len = te - q;
      double v;
      if (ord == 0) {                                            // the label: float(target)
        if (svm::parse_py_float(tok, len, &v) != svm::NUM_OK) code = ARB_LIBSVM_E_LABEL;
        else if (WRITE) store_label(y_out, v);
      } else if (ord == 1 && len >= 3 && tok[0] == 'q' && tok[1] == 'i' && tok[2] == 'd') {
        is_qid = true;                                           // features[0].startswith(b'qid'): split(b':', 1)
        long long k = 3;
        while (k < len && tok[k] != ':') ++k;
        if (k == len) {
          code = ARB_LIBSVM_E_QID;
        } else {
          int64_t qv = 0;
          const int st = svm::parse_py_int(tok + k + 1, len - k - 1, INT64_MIN, INT64_MAX, &qv);
          code = st == svm::NUM_OK ? 0 : st == svm::NUM_OVERFLOW ? ARB_LIBSVM_E_QID_OVERFLOW : ARB_LIBSVM_E_QID;
          qid = qv;
        }
      } else {                                                   // idx_s, value = token.split(b':', 1)
        long long k = 0;
        while (k < len && tok[k] != ':') ++k;
        if (k == len) {
          code = ARB_LIBSVM_E_NO_COLON;
        } else {
          int64_t iv = 0;
          const int st = svm::parse_py_int(tok, k, INT32_MIN, INT32_MAX, &iv);
          if (st == svm::NUM_SYNTAX) code = ARB_LIBSVM_E_INDEX;
          else if (st == svm::NUM_OVERFLOW) code = ARB_LIBSVM_E_INDEX_OVERFLOW;
          else if (iv < 0) code = ARB_LIBSVM_E_NEGATIVE;
          else idx = static_cast<int>(iv);
          if (!code) {
            const int pst = svm::parse_py_float(tok + k + 1, len - k - 1, &v);
            if (pst == svm::NUM_SYNTAX) code = ARB_LIBSVM_E_VALUE;
            else if (pst != svm::NUM_OK) code = ARB_LIBSVM_E_UNSUPPORTED;
            else if (WRITE) store_feature(xrow + (idx - shift), v);
          }
        }
      }
    }
    // the index of the previous feature token: the nearest start lane below, or the previous window's last
    const unsigned below = S & lt;
    const int src = below ? 31 - __clz(below) : lane;
    const int from_lane = __shfl_sync(0xffffffffu, idx, src);
    const int prev = below ? from_lane : prev_idx;
    if (me && !code && idx >= 0 && idx <= prev) code = ARB_LIBSVM_E_NOT_SORTED;
    // sklearn raises at the first failing token of the line
    const unsigned bad = __ballot_sync(0xffffffffu, me && code);
    if (bad) {
      r.status = __shfl_sync(0xffffffffu, code, __ffs(bad) - 1);
      return r;
    }
    const unsigned qmask = __ballot_sync(0xffffffffu, is_qid);
    if (qmask) {
      r.has_qid = true;
      r.qid = __shfl_sync(0xffffffffu, qid, __ffs(qmask) - 1);
    }
    int mn = idx >= 0 ? idx : 0x7fffffff, mx = idx;
    for (int o = 16; o; o >>= 1) {
      mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    r.min_idx = min(r.min_idx, mn);
    r.max_idx = max(r.max_idx, mx);
    const int last = __shfl_sync(0xffffffffu, idx, 31 - __clz(S));
    if (last >= 0) prev_idx = last;
    r.ntok += __popc(S);
  }
  return r;
}

__device__ __forceinline__ void line_span(const long long* line_end, long long n_nl, long long n_bytes,
                                          long long line, long long* beg, long long* end) {
  *beg = line ? line_end[line - 1] + 1 : 0;
  *end = line < n_nl ? line_end[line] : n_bytes;
}

__global__ void __launch_bounds__(SVM_WARPS * 32) pass1_kernel(const uint8_t* __restrict__ text, long long n_bytes,
                                                               const long long* __restrict__ line_end, long long n_nl,
                                                               long long n_lines, long long* __restrict__ line_row,
                                                               long long* __restrict__ line_qid,
                                                               long long* __restrict__ summary) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * SVM_WARPS;
  unsigned long long err = ~0ull;
  long long mn = 0x7fffffff, mx = -1, no_qid = 0;
  for (long long line = (long long)blockIdx.x * SVM_WARPS + (threadIdx.x >> 5); line < n_lines; line += warps) {
    long long beg, end;
    line_span(line_end, n_nl, n_bytes, line, &beg, &end);
    const LineScan r = scan_line<false, float>(text, beg, end, 0, nullptr, nullptr);
    if (lane == 0) {
      line_row[line] = r.ntok > 0 && !r.status;
      line_qid[line] = r.qid;
      if (r.status) {
        const unsigned long long key = ((unsigned long long)(line + 1) << 8) | unsigned(r.status);
        err = key < err ? key : err;
      } else if (r.ntok > 0) {
        no_qid += !r.has_qid;
        mn = min(mn, (long long)r.min_idx);
        mx = max(mx, (long long)r.max_idx);
      }
    }
  }
  if (lane == 0) {
    if (err != ~0ull) atomicMin(reinterpret_cast<unsigned long long*>(summary + SUM_ERROR), err);
    if (mn != 0x7fffffff) atomicMin(summary + SUM_MIN_INDEX, mn);
    if (mx >= 0) atomicMax(summary + SUM_MAX_INDEX, mx);
    if (no_qid) atomicAdd(reinterpret_cast<unsigned long long*>(summary + SUM_NO_QID), (unsigned long long)no_qid);
  }
}

__global__ void summary_init_kernel(long long* summary) {
  if (threadIdx.x < SUM_WORDS) {
    const long long init[SUM_WORDS] = {-1, 0x7fffffff, -1, 0, 0, 0, 0, 0};   // SUM_ERROR: ~0 as unsigned
    summary[threadIdx.x] = init[threadIdx.x];
  }
}

template <typename T>
__global__ void __launch_bounds__(SVM_WARPS * 32) pass2_kernel(const uint8_t* __restrict__ text, long long n_bytes,
                                                               const long long* __restrict__ line_end, long long n_nl,
                                                               long long n_lines, const long long* __restrict__ line_row,
                                                               const long long* __restrict__ line_qid, long long n_rows,
                                                               int shift, long long F, T* __restrict__ docs_x,
                                                               T* __restrict__ docs_y, long long* __restrict__ qids) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * SVM_WARPS;
  for (long long line = (long long)blockIdx.x * SVM_WARPS + (threadIdx.x >> 5); line < n_lines; line += warps) {
    const long long row = line_row[line];
    const long long next = line + 1 < n_lines ? line_row[line + 1] : n_rows;
    if (next == row) continue;                       // not a row
    T* xrow = docs_x + (size_t)row * F;
    for (long long c = lane; c < F; c += 32) xrow[c] = T(0);
    __syncwarp();
    long long beg, end;
    line_span(line_end, n_nl, n_bytes, line, &beg, &end);
    scan_line<true, T>(text, beg, end, shift, xrow, docs_y + row);
    if (lane == 0) qids[row] = line_qid[line];
  }
}

}  // namespace arb

using namespace arb;

static int line_grid(long long n_lines) {
  const long long want = (n_lines + SVM_WARPS - 1) / SVM_WARPS;
  const long long cap = (long long)sm_count() * 16;
  return int(want < cap ? (want > 0 ? want : 1) : cap);
}

extern "C" int64_t arb_libsvm_chunks(int64_t n_bytes) { return n_bytes > 0 ? (n_bytes + LF_CHUNK - 1) / LF_CHUNK : 0; }

extern "C" int32_t arb_libsvm_count_lines(const uint8_t* text, int64_t n_bytes, int64_t* chunk_counts, void* stream) {
  if (!text || !chunk_counts || n_bytes <= 0 || (reinterpret_cast<uintptr_t>(text) & 15u)) {
    arb_set_error("arb_libsvm_count_lines: null pointer, misaligned text or n_bytes <= 0");
    return ARB_E_INVALID_ARG;
  }
  const long long chunks = arb_libsvm_chunks(n_bytes);
  if (chunks > 0x7fffffffLL) {
    arb_set_error("arb_libsvm_count_lines: text too large");
    return ARB_E_UNSUPPORTED;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (int rc = launch(lf_count_kernel, dim3(unsigned(chunks)), dim3(LF_THREADS), 0, st, false, text,
                      (long long)n_bytes, reinterpret_cast<long long*>(chunk_counts)))
    return rc;
  return launch(exclusive_scan_kernel, dim3(1), dim3(SCAN_THREADS), 0, st, false,
                reinterpret_cast<long long*>(chunk_counts), chunks, reinterpret_cast<long long*>(chunk_counts + chunks));
}

extern "C" int32_t arb_libsvm_index_lines(const uint8_t* text, int64_t n_bytes, const int64_t* chunk_counts,
                                          int64_t* line_end, void* stream) {
  if (!text || !chunk_counts || !line_end || n_bytes <= 0 || (reinterpret_cast<uintptr_t>(text) & 15u)) {
    arb_set_error("arb_libsvm_index_lines: null pointer, misaligned text or n_bytes <= 0");
    return ARB_E_INVALID_ARG;
  }
  const long long chunks = arb_libsvm_chunks(n_bytes);
  if (chunks > 0x7fffffffLL) {
    arb_set_error("arb_libsvm_index_lines: text too large");
    return ARB_E_UNSUPPORTED;
  }
  return launch(lf_write_kernel, dim3(unsigned(chunks)), dim3(LF_THREADS), 0, static_cast<cudaStream_t>(stream), false,
                text, (long long)n_bytes, reinterpret_cast<const long long*>(chunk_counts),
                reinterpret_cast<long long*>(line_end));
}

extern "C" int32_t arb_libsvm_pass1(const uint8_t* text, int64_t n_bytes, const int64_t* line_end, int64_t n_newlines,
                                    int64_t n_lines, int64_t* line_row, int64_t* line_qid, int64_t* summary,
                                    void* stream) {
  if (!text || !line_row || !line_qid || !summary || n_bytes <= 0 || n_newlines < 0 || (n_newlines > 0 && !line_end) ||
      n_lines < n_newlines || n_lines > n_newlines + 1 || n_lines <= 0) {
    arb_set_error("arb_libsvm_pass1: null pointer or inconsistent sizes");
    return ARB_E_INVALID_ARG;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  long long* lr = reinterpret_cast<long long*>(line_row);
  long long* sm = reinterpret_cast<long long*>(summary);
  if (int rc = launch(summary_init_kernel, dim3(1), dim3(32), 0, st, false, sm)) return rc;
  if (int rc = launch(pass1_kernel, dim3(line_grid(n_lines)), dim3(SVM_WARPS * 32), 0, st, false, text,
                      (long long)n_bytes, reinterpret_cast<const long long*>(line_end), (long long)n_newlines,
                      (long long)n_lines, lr, reinterpret_cast<long long*>(line_qid), sm))
    return rc;
  return launch(exclusive_scan_kernel, dim3(1), dim3(SCAN_THREADS), 0, st, false, lr, (long long)n_lines,
                sm + SUM_ROWS);
}

template <typename T>
static int32_t pass2(const char* name, const uint8_t* text, int64_t n_bytes, const int64_t* line_end,
                     int64_t n_newlines, int64_t n_lines, const int64_t* line_row, const int64_t* line_qid,
                     int64_t n_rows, int32_t shift, int64_t n_features, T* docs_x, T* docs_y, int64_t* qids,
                     void* stream) {
  if (!text || !line_row || !line_qid || !docs_x || !docs_y || !qids || n_bytes <= 0 || n_newlines < 0 ||
      (n_newlines > 0 && !line_end) || n_lines < n_newlines || n_lines > n_newlines + 1 || n_lines <= 0 ||
      n_rows <= 0 || n_rows > n_lines || (shift != 0 && shift != 1) || n_features <= 0 ||
      n_features > ARB_LIBSVM_MAX_FEATURES) {
    char msg[96];
    snprintf(msg, sizeof msg, "%s: null pointer or inconsistent sizes", name);
    arb_set_error(msg);
    return ARB_E_INVALID_ARG;
  }
  return launch(pass2_kernel<T>, dim3(line_grid(n_lines)), dim3(SVM_WARPS * 32), 0, static_cast<cudaStream_t>(stream),
                false, text, (long long)n_bytes, reinterpret_cast<const long long*>(line_end), (long long)n_newlines,
                (long long)n_lines, reinterpret_cast<const long long*>(line_row),
                reinterpret_cast<const long long*>(line_qid), (long long)n_rows, (int)shift, (long long)n_features, docs_x,
                docs_y, reinterpret_cast<long long*>(qids));
}

extern "C" int32_t arb_libsvm_pass2(const uint8_t* text, int64_t n_bytes, const int64_t* line_end, int64_t n_newlines,
                                    int64_t n_lines, const int64_t* line_row, const int64_t* line_qid, int64_t n_rows,
                                    int32_t shift, int64_t n_features, float* docs_x, float* docs_y, int64_t* qids,
                                    void* stream) {
  return pass2("arb_libsvm_pass2", text, n_bytes, line_end, n_newlines, n_lines, line_row, line_qid, n_rows, shift,
               n_features, docs_x, docs_y, qids, stream);
}

extern "C" int32_t arb_libsvm_pass2_f64(const uint8_t* text, int64_t n_bytes, const int64_t* line_end,
                                        int64_t n_newlines, int64_t n_lines, const int64_t* line_row,
                                        const int64_t* line_qid, int64_t n_rows, int32_t shift, int64_t n_features,
                                        double* docs_x, double* docs_y, int64_t* qids, void* stream) {
  return pass2("arb_libsvm_pass2_f64", text, n_bytes, line_end, n_newlines, n_lines, line_row, line_qid, n_rows,
               shift, n_features, docs_x, docs_y, qids, stream);
}

extern "C" int32_t arb_libsvm_parse_numerals_host(const uint8_t* text_host, const int64_t* offsets_host, int64_t n,
                                                  int32_t kind, uint64_t* out_host, int32_t* status_host) {
  if (!text_host || !offsets_host || !out_host || !status_host || n < 0 || kind < 0 || kind > 3) {
    arb_set_error("arb_libsvm_parse_numerals_host: null pointer, n < 0 or unknown kind");
    return ARB_E_INVALID_ARG;
  }
  for (int64_t i = 0; i < n; ++i) {
    const uint8_t* s = text_host + offsets_host[i];
    const int64_t len = offsets_host[i + 1] - offsets_host[i];
    uint64_t out = 0;
    int st;
    if (kind <= 1) {
      double v = 0.0;
      st = svm::parse_py_float(s, len, &v);
      if (kind == 0) __builtin_memcpy(&out, &v, 8);
      else out = svm::sklearn_f32_bits(v, false);
    } else {
      int64_t iv = 0;
      st = kind == 2 ? svm::parse_py_int(s, len, INT32_MIN, INT32_MAX, &iv)
                     : svm::parse_py_int(s, len, INT64_MIN, INT64_MAX, &iv);
      out = static_cast<uint64_t>(iv);
    }
    out_host[i] = st == svm::NUM_OK ? out : 0;
    status_host[i] = st;
  }
  return ARB_OK;
}
