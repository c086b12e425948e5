// hhg_msa.cuh -- A3M multiple alignments -> HMMs on the device (SURVEY §8 rows a10 / f1: the A3M branch of
// HHEntry::getTemplateHMM, src/hhdatabase.cpp:441-449, and the query path Alignment -> HMM of hhblits).
//
//   host  : MsaScanner       -- Alignment::Read (src/hhalignment.cpp:181-544) + Compress with match states by case
//                               (M = 1, :889-990): residues -> X[k][i] codes, insert counts, first/last/nres, the
//                               length sort of Filter2 (:1673-1681, the reference's own quicksort, tie order kept)
//   device: k_msa_filter     -- Alignment::Filter2 (:1598-1968): coverage / qid / qsc tests and the greedy
//                               maximum-pairwise-identity filter, one thread block per alignment
//           k_msa_weights    -- global sequence weights wg (FrequenciesAndTransitions :2083-2108)
//           k_msa_mstate     -- position-specific weights on sub-alignments, emission frequencies, M->x transitions,
//                               Neff_M (Amino_acid_frequencies_and_transitions_from_M_state :2408-2683)
//           k_msa_finish     -- Neff_HMM, I->x / D->x transitions, Neff_I / Neff_D, end states (:2957-3382)
//           k_msa_prepare    -- the HHM loader's pseudocount step (hhg_hhm.cuh) fed with floats instead of file integers
//
// Arithmetic keeps the reference's types and order (float / double, unfused, sums in ascending sequence and column
// order).  ONE step of the reference is not portable arithmetic: the weight contribution 1/(n*naa) is taken with
// simdf32_rcp = RCPPS (:2531), an approximation whose bits differ between CPU vendors.  The library samples the
// host's own RCPPS for every possible argument (n*naa <= 65535*20, integers) at first use and the kernel looks the
// value up, so the result is bit-identical to the reference running on the same host.
#pragma once
#include <algorithm>
#include <cctype>
#include <cfloat>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "hhg_math.cuh"
#ifndef HHG_EMUL            // tests/emul compiles the kernels of this file for the CPU, without the CUDA-only headers
#include "hhg_hhm.cuh"
#include "hhg_kernels.cuh"
#endif

namespace hhg {

constexpr int MSA_ANY = 20, MSA_GAP = 21, MSA_ENDGAP = 22;   // src/hhdecl.h:52-56
constexpr int MSA_RCP_N = 1 << 21;                            // > 65535 * 20
constexpr int MSA_MSTATE_THREADS = 128;                       // block size of k_msa_mstate (see the kernel)
constexpr int MSA_TAIL = 32;                                  // bytes after column L+1 of a row: what Filter2 reads there

// ------------------------------------------------------------------------------------------ host: scanner
struct MsaHost {
  int N_in = 0, L = 0, stride = 0;
  int kfirst = -1, kss_dssp = -1, ksa_dssp = -1, kss_pred = -1, kss_conf = -1, N_ss = 0;
  std::vector<int8_t> keep, display;     // [N_in] as Alignment::Read leaves them (0 / 1 / 2); nres == 0 -> keep 0
  std::vector<uint8_t> X;                // [N_in][stride]: code 0..22 of columns 0..L+1, bit 7 = insert after the column,
                                         // then MSA_TAIL codes of columns L+1.. as Filter2 sees them (see compress)
  std::vector<int32_t> first, last, nres, ksort;   // [N_in]
  std::vector<uint32_t> ins_off;         // [L+2] CSR over columns 0..L of the inserts, ascending sequence index
  std::vector<int32_t> ins_k;
  std::vector<uint16_t> ins_cnt;
};

class MsaScanner {
 public:
  static int aa_code(char c) {           // aa2i, src/hhutil-inl.h:45-83
    if (c >= 'a' && c <= 'z') c = (char)(c + 'A' - 'a');
    switch (c) {
      case 'A': return 0; case 'R': return 1; case 'N': return 2; case 'D': return 3; case 'C': return 4;
      case 'Q': return 5; case 'E': return 6; case 'G': return 7; case 'H': return 8; case 'I': return 9;
      case 'L': return 10; case 'K': return 11; case 'M': return 12; case 'F': return 13; case 'P': return 14;
      case 'S': return 15; case 'T': return 16; case 'W': return 17; case 'Y': return 18; case 'V': return 19;
      case 'X': case 'J': case 'O': return MSA_ANY;
      case 'U': return 4; case 'B': return 3; case 'Z': return 6;
      case '-': case '.': case '_': return MSA_GAP;
    }
    if (c >= 0 && c <= 32) return -1;
    return -2;
  }
  static int ss_code(char c) {           // ss2i, src/hhutil-inl.h:123
    if (c >= 'a' && c <= 'z') c = (char)(c - 'a' + 'A');
    switch (c) {
      case '.': case '-': case 'X': return 0;
      case 'H': return 1; case 'E': return 2;
      case 'C': case '~': case 'I': return 3;
      case 'S': return 4; case 'T': return 5; case 'G': return 6; case 'B': return 7;
      case ' ': case '\t': case '\n': return -1;
      default: return -2;
    }
  }
  static char ss_canonical(char c) {     // ss2ss, src/hhutil-inl.h:217
    switch (c) {
      case '~': case 'I': return 'C';
      case 'i': return 'c';
      case 'H': case 'E': case 'C': case 'S': case 'T': case 'G': case 'B': case '.':
      case 'h': case 'e': case 'c': case 's': case 't': case 'g': case 'b': return c;
      default: return '-';
    }
  }
  static int sa_code(char c) {           // sa2i, src/hhutil-inl.h:173
    if (c >= 'a' && c <= 'z') c = (char)(c + 'A' - 'a');
    switch (c) {
      case '.': case '-': return 0;
      case 'A': return 1; case 'B': return 2; case 'C': return 3; case 'D': return 4; case 'E': return 5; case 'F': return 6;
      case ' ': case '\t': case '\n': return -1;
    }
    return -2;
  }
  static int cf_code(char c) {           // cf2i, src/hhutil-inl.h:248
    if (c >= '0' && c <= '9') return c - '0' + 1;
    return 0;
  }

  // Alignment::Read with mark == 0, then Compress with M == 1.  Returns "" or an error description (the cases in
  // which the reference exits).  maxseq / maxcol / maxres: Parameters of the same names (src/hhdecl.cpp:10-14).
  static std::string parse(const char* rec, int64_t len, int maxseq, int maxcol, int maxres, MsaHost* out, int M = 1,
                           int Mgaps = 50) {
    std::vector<std::string> seq;
    std::string msg = read_a3m(rec, len, maxseq, maxcol, out, &seq);
    if (!msg.empty()) return msg;
    return compress(seq, maxres, out, M, Mgaps);
  }

  // The sequence database of a compressed alignment database (`<db>_sequence.ffdata` + the offset / length columns of
  // its `.ffindex`, IN INDEX-FILE ORDER: ReadCompressed addresses entries with ffindex_get_entry_by_index).
  struct SeqDb { int64_t n; const char* data; const int64_t* off; const int64_t* len; };

  // Alignment::ReadCompressed (src/hhalignment.cpp:546-815) with mark == 0, then Compress with M == 1.
  static std::string parse_ca3m(const char* rec, int64_t len, const SeqDb& db, int maxseq, int maxcol, int maxres, MsaHost* out,
                                int M = 1, int Mgaps = 50) {
    std::vector<std::string> seq;
    std::string msg = read_ca3m(rec, len, db, maxseq, maxcol, out, &seq);
    if (!msg.empty()) return msg;
    return compress(seq, maxres, out, M, Mgaps);
  }

 private:
  static std::string read_ca3m(const char* rec, int64_t len, const SeqDb& db, int maxseq, int maxcol, MsaHost* out,
                               std::vector<std::string>* seq_out) {
    MsaHost& A = *out;
    A = MsaHost();
    std::vector<std::string>& seq = *seq_out;
    const int64_t data_size = len - 1;            // entry->length - 1: the ffindex entry ends with NUL
    int64_t ix = 0;
    const char* d = rec;
    if (data_size <= 0) return "empty record";
    if (d[0] == '#') {                            // name line
      ++ix;
      while (ix < data_size && isspace((unsigned char)d[ix])) ++ix;
      while (ix < data_size && d[ix] != '\n') ++ix;
      ++ix;
    }
    std::string header, cons;
    char last = '\0';
    int in_cons = 0;
    while (ix < data_size && !(last == '\n' && d[ix] == ';')) {
      if (d[ix] == '\n') ++in_cons;
      else if (in_cons == 0) header.push_back(d[ix]);
      else if (in_cons == 1) cons.push_back(d[ix]);
      last = d[ix];
      ++ix;
    }
    ++ix;                                         // past ';'
    if ((int)cons.size() > maxcol - 2) return "consensus longer than maxcol-2";
    const size_t consensus_length = cons.size();
    std::string s0;
    for (char c : cons) if (aa_code(c) >= 0) s0.push_back(c);
    if (s0.empty()) return "the consensus sequence contains no residues";
    seq.push_back(s0);
    A.keep.push_back(0); A.display.push_back(2);  // the consensus row is shown, not part of the profile
    A.kfirst = 0;
    while (ix < data_size) {
      if (ix + 8 > data_size) return "truncated sequence record";
      const unsigned char* u = (const unsigned char*)d + ix;
      const uint32_t entry = u[0] | (u[1] << 8) | (u[2] << 16) | ((uint32_t)u[3] << 24);
      const unsigned start_pos = u[4] | (u[5] << 8), nr_blocks = u[6] | (u[7] << 8);
      ix += 8;
      if ((int64_t)entry >= db.n) return "sequence entry " + std::to_string(entry) + " is not in the sequence database";
      const char* sd = db.data + db.off[entry];
      const int64_t sl = db.len[entry];
      std::string cur;
      size_t pos = start_pos, ali_len = 0;
      for (unsigned b = 0; b < nr_blocks; ++b) {
        if (ix + 2 > data_size) return "truncated block list";
        const unsigned nm = (unsigned char)d[ix];
        const int nid = (signed char)d[ix + 1];
        ix += 2;
        for (unsigned i = 0; i < nm; ++i) {
          if (pos < 1 || (int64_t)pos > sl) return "block list runs past the end of sequence entry " + std::to_string(entry);
          cur.push_back(sd[pos - 1]); ++pos; ++ali_len;
        }
        if (nid > 0) {
          for (int i = 0; i < nid; ++i) {
            if (pos < 1 || (int64_t)pos > sl) return "block list runs past the end of sequence entry " + std::to_string(entry);
            cur.push_back((char)tolower((unsigned char)sd[pos - 1])); ++pos;
          }
        } else {
          for (int i = 0; i < -nid; ++i) { cur.push_back('-'); ++ali_len; }
        }
        if ((int)cur.size() > maxcol - 2) return "sequence longer than maxcol-2";
      }
      while (ali_len < consensus_length) { cur.push_back('-'); ++ali_len; }
      if ((int)cur.size() > maxcol - 2) return "sequence longer than maxcol-2";
      std::string s;
      for (char c : cur) if (aa_code(c) >= 0) s.push_back(c);
      if ((int)seq.size() >= maxseq) return "more than maxseq sequences";
      seq.push_back(s);
      A.keep.push_back(1); A.display.push_back(1);
    }
    A.N_in = (int)seq.size();
    if (A.N_in - (A.keep[A.kfirst] == 0 ? 1 : 0) == 0) return "the alignment contains no master sequence";
    return "";
  }

  static std::string read_a3m(const char* rec, int64_t len, int maxseq, int maxcol, MsaHost* out,
                              std::vector<std::string>* seq_out) {
    MsaHost& A = *out;
    A = MsaHost();
    std::vector<std::string>& seq = *seq_out;
    const char* p = rec;
    const char* end = rec + len;
    { const void* z = memchr(rec, '\0', (size_t)len); if (z) end = (const char*)z; }   // ffindex entries end with NUL
    std::string cur;
    int k = -1;
    bool skip = false;
    auto flush = [&]() -> bool {         // "sequence ... contains no residues" (:224-228)
      if (k >= 0) { if (cur.empty()) return false; seq.push_back(cur); }
      return true;
    };
    bool stop = false;
    while (p < end && !stop) {
      const char* e = (const char*)memchr(p, '\n', (size_t)(end - p));
      if (!e) e = end;
      const char* next = e < end ? e + 1 : end;
      const size_t n = (size_t)(e - p);
      if (n > 0 && p[0] == '>') {
        if (k >= maxseq - 1) { stop = true; break; }        // "Maximum number of sequences exceeded": rest ignored
        if (!flush()) return "a sequence contains no residues";
        skip = false;
        ++k;
        cur.clear();
        A.keep.resize(k + 1); A.display.resize(k + 1);
        auto starts = [&](const char* s) { const size_t m = strlen(s); return n >= m && !memcmp(p, s, m); };
        auto special = [&](int& slot) {                     // first occurrence kept, later ones dropped (:264-309)
          if (slot < 0) { A.display[k] = 2; A.keep[k] = 0; slot = k; ++A.N_ss; return true; }
          skip = true; --k; A.keep.resize(k + 1); A.display.resize(k + 1); return false;
        };
        if (starts(">ss_dssp")) { if (!special(A.kss_dssp)) { p = next; continue; } }
        else if (starts(">sa_dssp")) { if (!special(A.ksa_dssp)) { p = next; continue; } }
        else if (starts(">ss_pred")) { if (!special(A.kss_pred)) { p = next; continue; } }
        else if (starts(">ss_conf")) { if (!special(A.kss_conf)) { p = next; continue; } }
        else if (starts(">ss_") || starts(">sa_")) { A.display[k] = 2; A.keep[k] = 0; ++A.N_ss; }
        else if (starts(">aa_")) { skip = true; --k; A.keep.resize(k + 1); A.display.resize(k + 1); p = next; continue; }
        else if (A.kfirst < 0) {
          // first word of the line (strwrd) containing "_consensus" -> not part of the profile (:322-334)
          const char* w = p;
          while (w < e && (unsigned char)*w <= 32) ++w;
          const char* we = w;
          while (we < e && (unsigned char)*we > 32) ++we;
          const std::string word(w, we);
          A.display[k] = 2;
          A.keep[k] = word.find("_consensus") != std::string::npos ? 0 : 2;
          A.kfirst = k;
        } else { A.display[k] = A.keep[k] = 1; }
      } else if (n > 0 && p[0] == '#') {
        // '#' line: name / longname only
      } else if (!skip) {
        if (k == -1) { p = next; continue; }               // "No sequence name preceding following line"
        const bool is_aa = A.keep[k] || k == A.kfirst;
        for (const char* h = p; h < e && (signed char)*h > 0 && (int)cur.size() < maxcol - 2; ++h) {
          const char c = *h;
          if (is_aa) { if (aa_code(c) >= 0) cur.push_back(c); }
          else if (k == A.kss_dssp) { const int s = ss_code(c); if (s >= 0 && s <= 7) cur.push_back(ss_canonical(c)); }
          else if (k == A.ksa_dssp) { if (sa_code(c) >= 0) cur.push_back(c); }
          else if (k == A.kss_pred) { const int s = ss_code(c); if (s >= 0 && s <= 3) cur.push_back(ss_canonical(c)); }
          else if (k == A.kss_conf) { if (c == '-' || c == '.' || (c >= '0' && c <= '9')) cur.push_back(c); }
          else if (A.display[k]) { if (c == '-' || c == '.' || (c >= '0' && c <= '9') || c == 'A' || c == 'B') cur.push_back(c); }
        }
        if ((int)cur.size() >= maxcol - 2) skip = true;    // "maximum number of residues exceeded": rest of it dropped
      }
      p = next;
    }
    if (k < 0) return "no sequences found";
    if (cur.empty()) return "a sequence contains no residues";
    seq.push_back(cur);
    A.N_in = k + 1;
    if ((int)seq.size() != A.N_in) return "internal: sequence count";
    if (A.kfirst < 0 || (A.N_in - A.N_ss - (A.keep[A.kfirst] == 0 ? 1 : 0)) == 0) return "the alignment contains no master sequence";
    return "";
  }

  static std::string compress(const std::vector<std::string>& seq, int maxres, MsaHost* out, int M = 1, int Mgaps = 50) {
    MsaHost& A = *out;

    // ---- Compress, case M == 1 (:889-990)
    const int N = A.N_in;
    std::vector<std::vector<uint8_t>> X(N);
    std::vector<std::vector<uint16_t>> I(N);
    int L = maxres - 2, unequal = 0;
    std::vector<int> raw_nres;                              // see the M == 2 branch
    std::vector<std::vector<uint8_t>> tail(N);              // see the M == 2 branch
    // "Too few match states" (:861-880): a file with ONE sequence whose upper-case letters + '-' number fewer than 6
    // is read as if -M first had been given: every letter of that sequence is a match state, '-' columns are not
    bool by_first = M == 3;
    if (M == 1 && N - A.N_ss <= 1) {
      int ms = 0;
      for (char c : seq[A.kfirst]) ms += (c >= 'A' && c <= 'Z') || c == '-';
      by_first = ms < 6;
    }
    if (M == 2) {                                           // Compress, case M == 2 (:994-1175): gap-percentage rule
      const size_t raw = seq[A.kfirst].size();
      for (int q = 0; q < N; ++q)
        if ((A.keep[q] || q == A.kss_dssp || q == A.kss_pred || q == A.ksa_dssp || q == A.kss_conf) && seq[q].size() != raw)
          return "sequences do not all have the same number of columns (sequence " + std::to_string(q) + ")";
      // residue codes of all columns, residues per row, quick sequence weights (:1012-1051)
      std::vector<std::vector<uint8_t>> C(N);
      std::vector<int> nr(N, 0);
      std::vector<float> wq(N, 0.f);
      for (int q = 0; q < N; ++q) {
        if (!A.keep[q]) continue;
        C[q].resize(raw);
        for (size_t l = 0; l < raw; ++l) { C[q][l] = (uint8_t)aa_code(seq[q][l]); nr[q] += C[q][l] < 20; }
      }
      for (size_t l = 0; l < raw; ++l) {
        int nl[23] = {0};
        for (int q = 0; q < N; ++q) if (A.keep[q]) ++nl[C[q][l]];
        int naa = 0;
        for (int a = 0; a < 20; ++a) naa += nl[a] != 0;
        if (!naa) naa = 1;
        for (int q = 0; q < N; ++q)
          if (A.keep[q] && C[q][l] < 20) wq[q] += 1.0 / float(nl[C[q][l]] * naa * (nr[q] + 30.0));
      }
      for (int q = 0; q < N; ++q) {                         // end gaps over the raw columns (:1054-1062)
        if (!A.keep[q]) continue;
        for (size_t l = 0; l < raw && C[q][l] == MSA_GAP; ++l) C[q][l] = MSA_ENDGAP;
        for (size_t l = raw; l-- > 0 && C[q][l] == MSA_GAP;) C[q][l] = MSA_ENDGAP;
      }
      for (int q = 0; q < N; ++q) { X[q].assign(1, MSA_ANY); I[q].assign(1, 0); }
      int i = 0, kfirst = A.kfirst;
      for (size_t l = 0; l < raw; ++l) {
        float res = 0, gap = 0;
        for (int q = 0; q < N; ++q) {
          if (!A.keep[q]) continue;
          if (C[q][l] < MSA_GAP) res += wq[q];
          else if (C[q][l] != MSA_ENDGAP) gap += wq[q];
        }
        const float pg = 100. * gap / (res + gap);
        if (pg <= float(Mgaps)) {
          if (i >= maxres - 2) break;
          ++i;
          for (int q = 0; q < N; ++q) {
            const char c = seq[q].size() > l ? seq[q][l] : '-';
            if (A.keep[q]) { X[q].push_back(C[q][l]); I[q].push_back(0); if (kfirst == -1) kfirst = q; }
            else if (q == A.kss_dssp || q == A.kss_pred) X[q].push_back((uint8_t)ss_code(c));
            else if (q == A.ksa_dssp) X[q].push_back((uint8_t)sa_code(c));
            else if (q == A.kss_conf) X[q].push_back((uint8_t)cf_code(c));
            else { X[q].push_back((uint8_t)MSA_GAP); if (q == kfirst) kfirst = -1; }   // a consensus master row drops out (:1131-1133)
          }
        } else {
          for (int q = 0; q < N; ++q) if (A.keep[q] && C[q][l] < MSA_GAP) ++I[q].back();
        }
      }
      if (kfirst < 0) return "the alignment contains no master sequence";
      A.kfirst = kfirst;
      L = i;
      // Compress moves the match columns to the front of each row in place, so beyond column L the rows still hold the
      // codes of input columns L+1, L+2, ... while Filter2 runs (FrequenciesAndTransitions sets X[k][L+1] = ENDGAP only
      // afterwards).  Filter2's 32-byte windows reach up to 31 columns past L and count residues found there.
      for (int q = 0; q < N; ++q)
        if (A.keep[q] && raw > (size_t)L) tail[q].assign(C[q].begin() + L, C[q].begin() + std::min(raw, (size_t)L + MSA_TAIL));
      // Compress fills nres[] with the residues over ALL input columns here, and Filter2 recomputes it over the match
      // columns only `if (nres == NULL || sizeof(nres) < N_in * sizeof(int))` (:1660), i.e. only when N_in > 2
      if (N <= 2) raw_nres = nr;
    } else if (by_first) {                                  // Compress, case M == 3 (:1178-1262)
      const size_t raw = seq[0].size();
      for (int q = 1; q < N; ++q) if (seq[q].size() != raw) return "sequences do not all have the same number of columns (sequence " + std::to_string(q) + ")";
      const std::string& fs = seq[A.kfirst];
      for (int q = 0; q < N; ++q) { X[q].assign(1, MSA_ANY); I[q].assign(1, 0); }
      int i = 0;
      for (size_t l = 0; l < raw; ++l) {
        if (isalpha((unsigned char)fs[l])) {
          if (i >= maxres - 2) break;
          ++i;
          for (int q = 0; q < N; ++q) {
            const char c = seq[q][l];
            if (A.keep[q]) { X[q].push_back((uint8_t)aa_code(c)); I[q].push_back(0); }
            else if (q == A.kss_dssp || q == A.kss_pred) X[q].push_back((uint8_t)ss_code(c));
            else if (q == A.ksa_dssp) X[q].push_back((uint8_t)sa_code(c));
            else if (q == A.kss_conf) X[q].push_back((uint8_t)cf_code(c));
            else X[q].push_back((uint8_t)MSA_GAP);         // rows the reference leaves at their initial GAP
          }
        } else {
          for (int q = 0; q < N; ++q) if (A.keep[q] && aa_code(seq[q][l]) < MSA_GAP) ++I[q].back();
        }
      }
      L = i;
    } else
    for (int q = 0; q < N; ++q) {
      const std::string& s = seq[q];
      std::vector<uint8_t>& x = X[q];
      std::vector<uint16_t>& in = I[q];
      x.assign(1, MSA_ANY);
      in.assign(1, 0);
      bool counted = true;
      if (A.keep[q]) {
        for (char c : s) {
          if (c >= 'a' && c <= 'z') ++in.back();
          else if (c != '.') { x.push_back((uint8_t)aa_code(c)); in.push_back(0); }
        }
      } else if (q == A.kss_dssp || q == A.kss_pred) {
        for (char c : s) if (c != '.' && !(c >= 'a' && c <= 'z')) x.push_back((uint8_t)ss_code(c));
      } else if (q == A.ksa_dssp) {
        for (char c : s) if (c != '.' && !(c >= 'a' && c <= 'z')) x.push_back((uint8_t)sa_code(c));
      } else if (q == A.kss_conf) {
        for (char c : s) if (c != '.') x.push_back((uint8_t)cf_code(c));
      } else if (q == A.kfirst) {
        for (char c : s) if (c != '.') { x.push_back((uint8_t)aa_code(c)); in.push_back(0); }
      } else counted = false;
      if (!counted) continue;
      const int i = (int)x.size() - 1;
      if (L != i && L != maxres - 2 && !unequal) unequal = q;
      L = L < i ? L : i;
    }
    if (unequal) return "sequences do not all have the same number of match columns (sequence " + std::to_string(unequal) + ")";
    if (L <= 0) return "the alignment contains no match states";
    if (L == maxres - 2) return "more than maxres-2 match columns";
    A.L = L;
    A.stride = (L + 2 + MSA_TAIL + 3) & ~3;
    A.X.assign((size_t)N * A.stride, (uint8_t)MSA_GAP);      // initX: rows are GAP beyond what was written
    A.ins_off.assign((size_t)L + 2, 0);
    for (int q = 0; q < N; ++q) {
      uint8_t* row = A.X.data() + (size_t)q * A.stride;
      const std::vector<uint8_t>& x = X[q];
      for (int i = 0; i < (int)x.size() && i <= L + 1; ++i) row[i] = x[i];
      row[0] = MSA_ANY;
      if (A.keep[q] && M != 2) {                            // end gaps (:969-977; with M == 2 they were marked on the raw columns)
        for (int i = 1; i <= L && row[i] == MSA_GAP; ++i) row[i] = MSA_ENDGAP;
        for (int i = L; i >= 1 && row[i] == MSA_GAP; --i) row[i] = MSA_ENDGAP;
      }
      // FrequenciesAndTransitions sets X[k][0] = X[k][L+1] = ENDGAP before the weighting (:2103-2106); neither column
      // takes part in Filter2 (both codes are "no residue"), so column L+1 carries ENDGAP from the start and column 0
      // is never read as a predecessor (k_msa_mstate treats it as "not in the sub-alignment")
      row[L + 1] = MSA_ENDGAP;
      std::copy(tail[q].begin(), tail[q].end(), row + L + 2);  // GAP where the reference's row holds no residue there
    }
    // first / last / nres over ALL rows, nres == 0 -> keep 0 (Filter2 :1647-1676)
    A.first.resize(N); A.last.resize(N); A.nres.resize(N); A.ksort.resize(N);
    for (int q = 0; q < N; ++q) {
      const uint8_t* row = A.X.data() + (size_t)q * A.stride;
      int i;
      for (i = 1; i <= L; ++i) if (row[i] < 20) break;
      A.first[q] = i;
      for (i = L; i >= 1; --i) if (row[i] < 20) break;
      A.last[q] = i;
      int nr = 0;
      for (i = A.first[q]; i <= A.last[q]; ++i) if (row[i] < 20) ++nr;
      if (!raw_nres.empty()) { A.nres[q] = A.keep[q] ? raw_nres[q] : 0; A.ksort[q] = q; continue; }
      A.nres[q] = nr;
      if (nr == 0) A.keep[q] = 0;
      A.ksort[q] = q;
    }
    qsort_desc(A.nres.data(), A.ksort.data(), A.kfirst + 1, N - 1);
    // inserts: bit 7 of the column byte + CSR by column (rows that enter the profile, or the master row)
    for (int q = 0; q < N; ++q) {
      if (!(A.keep[q] || q == A.kfirst)) continue;
      const std::vector<uint16_t>& in = I[q];
      for (int i = 0; i <= L && i < (int)in.size(); ++i) if (in[i]) ++A.ins_off[i + 1];
    }
    for (int i = 0; i <= L; ++i) A.ins_off[i + 1] += A.ins_off[i];
    A.ins_k.resize(A.ins_off[L + 1]); A.ins_cnt.resize(A.ins_off[L + 1]);
    std::vector<uint32_t> fill(A.ins_off.begin(), A.ins_off.end() - 1);
    for (int q = 0; q < N; ++q) {
      if (!(A.keep[q] || q == A.kfirst)) continue;
      const std::vector<uint16_t>& in = I[q];
      uint8_t* row = A.X.data() + (size_t)q * A.stride;
      for (int i = 0; i <= L && i < (int)in.size(); ++i)
        if (in[i]) { A.ins_k[fill[i]] = q; A.ins_cnt[fill[i]] = in[i]; ++fill[i]; row[i] |= 0x80; }
    }
    return "";
  }

  // QSortInt(v, k, left, right, -1), src/util.cpp:247-274, with an explicit stack (same swap sequence)
  static void qsort_desc(const int* v, int* k, int left, int right) {
    std::vector<std::pair<int, int>> st;
    st.emplace_back(left, right);
    while (!st.empty()) {
      const int l = st.back().first, r = st.back().second;
      st.pop_back();
      if (l >= r) continue;
      std::swap(k[l], k[(l + r) / 2]);
      int last = l;
      for (int i = l + 1; i <= r; ++i)
        if (v[k[i]] > v[k[l]]) { ++last; std::swap(k[last], k[i]); }
      std::swap(k[l], k[last]);
      st.emplace_back(last + 1, r);      // popped second: the reference sorts the left part first; the parts are disjoint
      st.emplace_back(l, last - 1);
    }
  }
};

// ------------------------------------------------------------------------------------------ device
struct MsaDesc {           // one alignment of a chunk
  int N, L, stride, kfirst;
  long long x_off;         // bytes into X
  long long seq_off;       // per-sequence arrays
  long long col_off;       // per-column arrays with L+2 entries per alignment
  long long ins_base;      // inserts
};

struct MsaFilterParams {   // Alignment::Filter arguments
  int max_seqid, coverage, qid, Ndiff;
  float qsc;
  float S[400];            // substitution matrix in bits (qsc test)
};

struct MsaArrays {
  const MsaDesc* desc;
  const uint8_t* X;
  int8_t* keep;            // in: after Read/Compress; out: after Filter2
  const int8_t* display;
  const int* first; const int* last; const int* nres; const int* ksort;
  int* in_; int* inkk; int* seqid_prev; int* acc;     // [seq]
  int* Ncnt; int* Nmax; int* idmaxwin;                // [col]
  float* wg;                                          // [seq]
  const uint32_t* ins_off; const int* ins_k; const uint16_t* ins_cnt;
  int* n_filtered;         // [m]
  int* status;             // [m] 0 ok, else an error code
  float* f; float* tr; float* neff_m; float* neff_i; float* neff_d; float* neff_seg;   // outputs, [col]
  float* neff_hmm;         // [m]
};

__device__ __forceinline__ int msa_x(const uint8_t* row, int i) { return row[i] & 0x7f; }

// ---- Filter2 ---------------------------------------------------------------------------------------------------
// One block per alignment.  The control flow of the reference is executed by every thread on block-shared state; the
// O(N^2 L) part -- does ANY already accepted longer sequence j make candidate k redundant -- runs warp per pair.
// The pairwise test (:1884-1923) counts, over the columns where both rows hold a residue, the columns that differ;
// the reference's 32-byte SIMD windows and its early exit change neither count when the test can still reject.
__global__ void __launch_bounds__(256)
k_msa_filter(MsaArrays A, const __grid_constant__ MsaFilterParams P) {
  const MsaDesc d = A.desc[blockIdx.x];
  const int N = d.N, L = d.L, tid = threadIdx.x, T = blockDim.x;
  const uint8_t* X = A.X + d.x_off;
  int8_t* keep = A.keep + d.seq_off;
  const int8_t* display = A.display + d.seq_off;
  const int* first = A.first + d.seq_off; const int* last = A.last + d.seq_off;
  const int* nres = A.nres + d.seq_off; const int* ksort = A.ksort + d.seq_off;
  int* in_ = A.in_ + d.seq_off; int* inkk = A.inkk + d.seq_off; int* seqid_prev = A.seqid_prev + d.seq_off;
  int* acc = A.acc + d.seq_off;
  int* Nc = A.Ncnt + d.col_off; int* Nmax = A.Nmax + d.col_off; int* idw = A.idmaxwin + d.col_off;
  const int kfirst = d.kfirst;
  const int WFIL = 25;
  __shared__ int s_n, s_flag, s_max, s_min, s_nacc, s_red[8];

  if (tid == 0) { s_n = 0; s_nacc = 0; }
  __syncthreads();
  int cnt = 0;
  for (int k = tid; k < N; k += T) {
    const int two = keep[k] == 2;
    in_[k] = two ? 2 : 0;
    cnt += two;
    seqid_prev[k] = -1;
  }
  if (cnt) atomicAdd(&s_n, cnt);
  for (int i = 1 + tid; i <= L; i += T) {
    Nc[i] = (i >= first[kfirst] && i <= last[kfirst]) ? 1 : 0;
    Nmax[i] = 0;
    idw[i] = -1;
  }
  int seqid1 = 20, seqid2 = P.max_seqid, Ndiff = P.Ndiff;
  if (Ndiff <= 0 || Ndiff >= N) { seqid1 = seqid2; Ndiff = N; }
  int diffNmax = Ndiff, diffNmax_prev = 0;
  __syncthreads();

  // coverage, score per column with the master row, identity with the master row (:1712-1772)
  const float qdiff_max_frac = __double2float_rn(0.9999 - 0.01 * (double)P.qid);
  const uint8_t* XQ = X + (size_t)kfirst * d.stride;
  for (int k = tid; k < N; k += T) {
    if (keep[k] == 0 || keep[k] == 2) continue;
    if (100 * nres[k] < P.coverage * L) { keep[k] = 0; continue; }
    const uint8_t* XK = X + (size_t)k * d.stride;
    if (P.qsc > -10.f) {
      const float qsc_min = __fmul_rn(P.qsc, (float)nres[k]);
      float sum = 0.f;
      int gapq = 0, gapk = 0;
      for (int i = first[k]; i <= last[k]; ++i) {
        const int xk = msa_x(XK, i), xq = msa_x(XQ, i);
        if (xk < 20) {
          gapk = 0;
          if (xq < 20) { gapq = 0; sum = __fadd_rn(sum, P.S[xq * 20 + xk]); }
          else if (xq == MSA_ANY) continue;
          else if (gapq++) sum = __fsub_rn(sum, 1.0f);
          else sum = __fsub_rn(sum, 6.0f);
        } else if (xk == MSA_ANY) continue;
        else if (xq < 20) {
          gapq = 0;
          if (gapk++) sum = __fsub_rn(sum, 1.0f);
          else sum = __fsub_rn(sum, 6.0f);
        }
      }
      if (sum < qsc_min) { keep[k] = 0; continue; }
    }
    if (qdiff_max_frac < 0.999f) {
      const int qdiff_max = (int)((double)__fmul_rn(qdiff_max_frac, (float)nres[k]) + 0.9999);
      int diff = 0;
      for (int i = first[k]; i <= last[k]; ++i) {
        const int xk = msa_x(XK, i);
        if (xk < 20 && xk != msa_x(XQ, i) && ++diff >= qdiff_max) break;
      }
      if (diff >= qdiff_max) { keep[k] = 0; continue; }
    }
  }
  __syncthreads();
  // "If no sequence left ... put back first real sequence" (:1775-1809)
  if (tid == 0) s_flag = 0;
  __syncthreads();
  cnt = 0;
  for (int k = tid; k < N; k += T) cnt += keep[k] > 0;
  if (cnt) atomicAdd(&s_flag, cnt);
  __syncthreads();
  const int nn = s_flag;
  __syncthreads();
  if (nn == 0 && tid == 0) {
    int k = 0;
    for (; k < N; ++k) if (display[k] != 2) { keep[k] = 1; break; }
    if (k >= N && display[kfirst] != 2) A.status[blockIdx.x] = 1;     // "does not contain any sequences"
  }
  __syncthreads();
  if (seqid1 > seqid2) {                 // (:1811-1813) returns before keep[] is replaced by in[]
    if (tid == 0) A.n_filtered[blockIdx.x] = nn;
    return;
  }
  for (int kk = tid; kk < N; kk += T) inkk[kk] = in_[ksort[kk]];
  __syncthreads();
  if (tid == 0) { int na = 0; for (int kk = 0; kk < N; ++kk) if (inkk[kk]) acc[na++] = kk; s_nacc = na; }
  __syncthreads();

  int seqid = seqid1, seqid_step = 0;
  while (seqid <= seqid2) {
    // position-dependent thresholds (:1821-1841)
    if (tid == 0) { s_flag = 1; s_max = 0; s_min = 0x7fffffff; s_red[0] = -0x7fffffff; }
    __syncthreads();
    diffNmax_prev = diffNmax;
    for (int i = 1 + tid; i <= L; i += T) {
      int mx = 0;
      const int j0 = max(1, min(L - 2 * WFIL + 1, i - WFIL)), j1 = min(L, max(2 * WFIL, i + WFIL));
      for (int j = j0; j <= j1; ++j) mx = max(mx, Nc[j]);
      int nm = Nmax[i];
      if (nm < mx) { nm = mx; Nmax[i] = nm; }
      if (nm < Ndiff) {
        atomicExch(&s_flag, 0);
        idw[i] = seqid;
        atomicMax(&s_max, Ndiff - nm);
      }
    }
    __syncthreads();
    // Nc is read above and written below: the window phase must be complete (barrier above)
    diffNmax = s_max;
    const int stop = s_flag;
    for (int i = 1 + tid; i <= L; i += T) { atomicMin(&s_min, idw[i]); atomicMax(&s_red[0], idw[i]); }
    __syncthreads();
    const int idw_min = s_min, idw_max = s_red[0];
    __syncthreads();
    if (stop) break;

    for (int kk = 0; kk < N; ++kk) {
      if (inkk[kk]) continue;
      const int k = ksort[kk];
      const int kp = keep[k];
      if (!kp) continue;
      if (kp == 2) { __syncthreads(); if (tid == 0) inkk[kk] = 2; __syncthreads(); continue; }
      if (seqid >= 100) {
        __syncthreads();
        if (tid == 0) { in_[k] = inkk[kk] = 1; ++s_n; acc[s_nacc++] = kk; }
        __syncthreads();
        continue;
      }
      const int fk = first[k], lk = last[k];
      int idm;
      if (idw_min == idw_max) idm = (fk <= lk) ? idw_max : -0x7fffffff;
      else {
        __syncthreads();
        if (tid == 0) s_max = -0x7fffffff;
        __syncthreads();
        int mx = -0x7fffffff;
        for (int i = fk + tid; i <= lk; i += T) mx = max(mx, idw[i]);
        if (mx > -0x7fffffff) atomicMax(&s_max, mx);
        __syncthreads();
        idm = s_max;
      }
      float seqidk = (float)seqid1;
      if ((float)idm > seqidk) seqidk = (float)idm;
      if (seqid == seqid_prev[k]) continue;
      __syncthreads();                   // every thread has read seqid_prev[k] and the flags of this candidate
      if (tid == 0) { seqid_prev[k] = seqid; s_flag = 0; }
      __syncthreads();
      const float dmf = __double2float_rn(0.9999 - 0.01 * (double)seqidk);
      const uint8_t* XK = X + (size_t)k * d.stride;
      const int nk = nres[k];
      const int nacc = s_nacc, warp = tid >> 5, lane = tid & 31, nw = T >> 5;
      for (int a = warp; a < nacc; a += nw) {
        // early exit once another warp has found a rejecting sequence; the decision must be warp-uniform (the lanes
        // meet again in the shuffles below), so one lane reads the flag for all
        int seen = lane == 0 ? atomicOr(&s_flag, 0) : 0;       // atomic on both sides: concurrent with the store below
        seen = __shfl_sync(0xffffffffu, seen, 0);
        if (seen) break;
        const int jj = acc[a];
        if (jj >= kk) continue;          // only longer (earlier in the sort) accepted sequences
        const int j = ksort[jj];
        const int f_kj = max(fk, first[j]), l_kj = min(lk, last[j]);
        const int cov0 = l_kj - f_kj + 1;
        const int diff_suff = (int)((double)__fmul_rn(dmf, (float)min(nk, cov0)) + 0.999);
        if (diff_suff <= 0) continue;    // the reference's loop body never runs: no rejection
        const uint8_t* XJ = X + (size_t)j * d.stride;
        int diff = 0, cov = 0;
        for (int w = (f_kj & ~3) + 4 * lane; w <= l_kj; w += 128) {
          const uint32_t a4 = *reinterpret_cast<const uint32_t*>(XK + w) & 0x7f7f7f7fu;
          const uint32_t b4 = *reinterpret_cast<const uint32_t*>(XJ + w) & 0x7f7f7f7fu;
          uint32_t both = __vcmpltu4(a4, 0x14141414u) & __vcmpltu4(b4, 0x14141414u);
          if (w + 3 > L) both &= (1u << 8 * (L + 1 - w)) - 1u;   // bytes past column L: the tail below
          const uint32_t ne = ~__vcmpeq4(a4, b4);
          cov += __popc(both) >> 3;
          diff += __popc(both & ne) >> 3;
        }
        // the reference's last window ends at the next multiple of 32 after l_kj; past column L it reads what Compress
        // left in the rows (input columns with -M <percent>, GAP otherwise), stored after column L+1 of each row
        if (lane < (l_kj / 32 + 1) * 32 - 1 - L) {
          const int a = XK[L + 2 + lane] & 0x7f, b = XJ[L + 2 + lane] & 0x7f;
          if (a < 20 && b < 20) { ++cov; diff += a != b; }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) { diff += __shfl_xor_sync(0xffffffffu, diff, o); cov += __shfl_xor_sync(0xffffffffu, cov, o); }
        if (lane == 0 && diff < diff_suff && (float)diff < __fmul_rn(dmf, (float)cov)) atomicExch(&s_flag, 1);
      }
      __syncthreads();
      const int rejected = s_flag;
      if (!rejected) {
        for (int i = fk + tid; i <= lk; i += T) ++Nc[i];
        if (tid == 0) { in_[k] = inkk[kk] = 1; ++s_n; acc[s_nacc++] = kk; }
      }
      __syncthreads();
    }
    const int den = diffNmax_prev - diffNmax + 1;
    if (den == 0) { if (tid == 0) A.status[blockIdx.x] = 2; break; }   // the reference would divide by zero here
    seqid_step = max(1, min(5, diffNmax / den * seqid_step / 2));
    seqid += seqid_step;
  }
  __syncthreads();
  for (int k = tid; k < N; k += T) keep[k] = (int8_t)in_[k];
  if (tid == 0) A.n_filtered[blockIdx.x] = s_n;
}

// ---- global weights (:2083-2108) --------------------------------------------------------------------------------
// Block per alignment.  scratch: ni[(L+2)*21] ints per alignment at col_off*21 (entry 20 = naa).
__global__ void __launch_bounds__(256)
k_msa_weights(MsaArrays A, int* __restrict__ ni_all) {
  const MsaDesc d = A.desc[blockIdx.x];
  const int N = d.N, L = d.L, tid = threadIdx.x, T = blockDim.x;
  const uint8_t* X = A.X + d.x_off;
  const int8_t* in = A.keep + d.seq_off;
  const int* nres = A.nres + d.seq_off;
  float* wg = A.wg + d.seq_off;
  int* ni = ni_all + d.col_off * 21;
  __shared__ unsigned short s_cnt[20][256];
  for (int i0 = 1; i0 <= L; i0 += T) {
    const int i = i0 + tid;
#pragma unroll
    for (int a = 0; a < 20; ++a) s_cnt[a][tid] = 0;
    if (i <= L) {
      for (int k = 0; k < N; ++k) {
        if (!in[k]) continue;
        const int x = msa_x(X + (size_t)k * d.stride, i);
        if (x < 20) ++s_cnt[x][tid];
      }
      int naa = 0;
#pragma unroll
      for (int a = 0; a < 20; ++a) { const int c = s_cnt[a][tid]; ni[(size_t)i * 21 + a] = c; naa += c != 0; }
      ni[(size_t)i * 21 + 20] = naa ? naa : 1;
    }
  }
  __syncthreads();
  for (int k = tid; k < N; k += T) {
    float w = 1e-6f;
    if (in[k]) {
      const uint8_t* row = X + (size_t)k * d.stride;
      const double len30 = (double)nres[k] + 30.0;
      for (int i = 1; i <= L; ++i) {
        const int x = msa_x(row, i);
        if (x < 20) {
          const float den = __double2float_rn(__dmul_rn((double)(ni[(size_t)i * 21 + x] * ni[(size_t)i * 21 + 20]), len30));
          w = __double2float_rn(__dadd_rn((double)w, __ddiv_rn(1.0, (double)den)));
        }
      }
    }
    wg[k] = w;
  }
  __syncthreads();
  __shared__ float s_fac;
  if (tid == 0) {                          // NormalizeTo1(wg, N_in), src/util-inl.h:277
    float sum = 0.f;
    for (int k = 0; k < N; ++k) sum = __fadd_rn(sum, wg[k]);
    s_fac = sum != 0.f ? __double2float_rn(__ddiv_rn(1.0, (double)sum)) : 1.0f;
    if (sum == 0.f) s_fac = 1.0f;
  }
  __syncthreads();
  const float fac = s_fac;
  for (int k = tid; k < N; k += T) wg[k] = __fmul_rn(wg[k], fac);
}

// ---- M state (:2408-2683), local weights ------------------------------------------------------------------------
// Persistent blocks pull (alignment, column) items; the block of a column at which the set of sequences with a
// residue changes owns the whole run of columns up to the next change: it builds the sub-alignment counts n[j][a],
// the weights wi[k], Neff of the run, and then the emission frequencies and M->x transitions of every column of the run.
// Block size: most of a block's time is ordered (single-thread or thread-per-row) work between barriers, so many small
// blocks beat few large ones: 128 threads, 16 KB of shared memory, 40 registers -> 12 resident blocks per SM.
__global__ void __launch_bounds__(MSA_MSTATE_THREADS)
k_msa_mstate(MsaArrays A, int n_msa, const long long* __restrict__ item_off, long long n_items, int* __restrict__ counter,
             int* __restrict__ cnt_all, float* __restrict__ wc_all, float* __restrict__ wi_all, uint8_t* __restrict__ mem_all,
             int Lmax, int Nmax_, const float* __restrict__ rcp, const float* __restrict__ pb, int use_global_weights,
             const float* __restrict__ lg2, const float* __restrict__ dif) {
  const int tid = threadIdx.x, T = blockDim.x, lane = tid & 31, warp = tid >> 5, nw = T >> 5;
  int* cnt = cnt_all + (size_t)blockIdx.x * (Lmax + 2) * 24;
  float* wc = wc_all + (size_t)blockIdx.x * (Lmax + 2) * 24;
  float* wi = wi_all + (size_t)blockIdx.x * Nmax_;
  uint8_t* member = mem_all + (size_t)blockIdx.x * Nmax_;
  __shared__ unsigned short s_cnt[23][MSA_MSTATE_THREADS];
  __shared__ float s_f[20][MSA_MSTATE_THREADS];
  __shared__ int s_item, s_any, s_nseq, s_jmin, s_jmax;
  __shared__ float s_neff;

  for (;;) {
    __syncthreads();
    if (tid == 0) s_item = atomicAdd(counter, 1);
    __syncthreads();
    const long long item = s_item;
    if (item >= n_items) return;
    int lo = 0, hi = n_msa - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (item_off[mid] <= item) lo = mid; else hi = mid - 1; }
    const MsaDesc d = A.desc[lo];
    const int i0 = (int)(item - item_off[lo]) + 1;
    const int N = d.N, L = d.L;
    if (A.n_filtered[lo] <= 1) continue;                   // single-sequence branch: k_msa_finish
    const uint8_t* X = A.X + d.x_off;
    const int8_t* in = A.keep + d.seq_off;
    const float* wg = A.wg + d.seq_off;
    float* F = A.f + d.col_off * 20;
    float* TR = A.tr + d.col_off * 7;
    float* NEFF = A.neff_seg + d.col_off;

    // does the set {k: in[k], residue in column i} differ between i0-1 and i0?  (column 0 counts as ENDGAP, :2104)
    auto changed = [&](int i) {
      __syncthreads();
      if (tid == 0) s_any = 0;
      __syncthreads();
      int any = 0;
      for (int k = tid; k < N; k += T) {
        if (!in[k]) continue;
        const uint8_t* row = X + (size_t)k * d.stride;
        const bool prev = i > 1 && msa_x(row, i - 1) < MSA_ANY, cur = msa_x(row, i) < MSA_ANY;
        any |= prev != cur;
      }
      if (any) atomicExch(&s_any, 1);
      __syncthreads();
      return s_any;
    };
    if (use_global_weights) {
      // wi = wg everywhere; every column is its own item
      for (int k = tid; k < N; k += T) wi[k] = wg[k];
    } else {
      if (!changed(i0)) {
        if (i0 > 1) continue;                              // interior of a run: its first column's block does it
        // i0 == 1 and no sequence has a residue there: Neff[1] = Neff[0] = 0, weights unused (all rows are gaps)
        for (int k = tid; k < N; k += T) wi[k] = 0.f;
        if (tid == 0) s_neff = 0.f;
        __syncthreads();
      } else {
        // ---- members, counts n[j][a] of the sub-alignment
        if (tid == 0) s_nseq = 0;
        __syncthreads();
        int c = 0;
        for (int k = tid; k < N; k += T) {
          const int mbr = in[k] && msa_x(X + (size_t)k * d.stride, i0) < MSA_ANY;
          member[k] = (uint8_t)mbr;
          c += mbr;
        }
        if (c) atomicAdd(&s_nseq, c);
        __syncthreads();
        const int nseqi = s_nseq;
        for (int j0 = 1; j0 <= L; j0 += T) {
          const int j = j0 + tid;
#pragma unroll
          for (int a = 0; a < 23; ++a) s_cnt[a][tid] = 0;
          if (j <= L) {
            for (int k = 0; k < N; ++k) {
              if (!member[k]) continue;
              ++s_cnt[msa_x(X + (size_t)k * d.stride, j)][tid];
            }
#pragma unroll
            for (int a = 0; a < 23; ++a) cnt[(size_t)j * 24 + a] = s_cnt[a][tid];
          }
        }
        // ---- columns with at most MAXENDGAPFRAC end gaps: jmin..jmax
        if (tid == 0) { s_jmin = L + 1; s_jmax = 0; }
        __syncthreads();
        const float thr = __fmul_rn(0.1f, (float)nseqi);
        for (int j = 1 + tid; j <= L; j += T) {
          if (!((float)cnt[(size_t)j * 24 + MSA_ENDGAP] > thr)) { atomicMin(&s_jmin, j); atomicMax(&s_jmax, j); }
        }
        __syncthreads();
        const int jmin = s_jmin, jmax = s_jmax;
        const int ncol = jmax - jmin + 1;
        if (ncol < 10) {                                     // NCOLMIN: global weights
          for (int k = tid; k < N; k += T) wi[k] = member[k] ? wg[k] : 0.0f;
        } else {
          for (int j = jmin + tid; j <= jmax; j += T) {
            int naa = 0;
#pragma unroll
            for (int a = 0; a < 20; ++a) naa += cnt[(size_t)j * 24 + a] != 0;
#pragma unroll
            for (int a = 0; a < 20; ++a) wc[(size_t)j * 24 + a] = rcp[cnt[(size_t)j * 24 + a] * naa];
            wc[(size_t)j * 24 + 20] = 0.f; wc[(size_t)j * 24 + 21] = 0.f; wc[(size_t)j * 24 + 22] = 0.f;
          }
          __syncthreads();
          for (int k = tid; k < N; k += T) {
            float w = 1e-8f;
            if (member[k]) {
              const uint8_t* row = X + (size_t)k * d.stride;
              for (int j = jmin; j <= jmax; ++j) w = __fadd_rn(w, wc[(size_t)j * 24 + msa_x(row, j)]);
            }
            wi[k] = w;
          }
        }
        __syncthreads();
        // ---- Neff of the run: entropy of the weighted columns jmin..jmax
        for (int j0 = jmin; j0 <= jmax; j0 += T) {
          const int j = j0 + tid;
#pragma unroll
          for (int a = 0; a < 20; ++a) s_f[a][tid] = 0.f;
          if (j <= jmax) {
            for (int k = 0; k < N; ++k) {
              if (!member[k]) continue;
              const int x = msa_x(X + (size_t)k * d.stride, j);
              if (x < 20) s_f[x][tid] = __fadd_rn(s_f[x][tid], wi[k]);
            }
            float sum = 0.f;
#pragma unroll
            for (int a = 0; a < 20; ++a) sum = __fadd_rn(sum, s_f[a][tid]);
            const float fac = sum != 0.f ? __double2float_rn(__ddiv_rn(1.0, (double)sum)) : 1.f;
#pragma unroll
            for (int a = 0; a < 20; ++a) {
              const float v = sum != 0.f ? __fmul_rn(s_f[a][tid], fac) : s_f[a][tid];
              wc[(size_t)j * 24 + a] = (double)v > 1E-10 ? __fmul_rn(v, fast_log2_dev(v, lg2, dif)) : 0.f;
            }
          }
        }
        __syncthreads();
        if (tid == 0) {
          float ne = 0.f;
          for (int j = jmin; j <= jmax; ++j) {
            const float4* t4 = reinterpret_cast<const float4*>(wc + (size_t)j * 24);
#pragma unroll
            for (int q = 0; q < 5; ++q) {
              const float4 v = t4[q];
              ne = __fsub_rn(ne, v.x); ne = __fsub_rn(ne, v.y); ne = __fsub_rn(ne, v.z); ne = __fsub_rn(ne, v.w);
            }
          }
          s_neff = ncol > 0 ? fpow2_dev(__fdiv_rn(ne, (float)ncol)) : 1.0f;
        }
        __syncthreads();
      }
    }
    // ---- the columns of the run: frequencies and M->x transitions, one warp per column
    const float neff_run = use_global_weights ? 0.f : s_neff;
    int iend = i0 + 1;                   // exclusive end of the run: the next column at which the set changes
    if (!use_global_weights) { while (iend <= L && !changed(iend)) ++iend; }
    __syncthreads();
    for (int c = i0 + warp; c < iend; c += nw) {
      float accv = 0.f;
      for (int k = 0; k < N; ++k) {
        if (!in[k]) continue;
        const uint8_t* row = X + (size_t)k * d.stride;
        const int xb = row[c], x = xb & 0x7f, xn = row[c + 1] & 0x7f;
        bool hit;
        if (lane < 20) hit = x == lane;
        else if (lane == 20) hit = x < MSA_ANY && (xb & 0x80);                                  // M -> I
        else if (lane == 21) hit = x < MSA_ANY && !(xb & 0x80) && xn <= MSA_ANY;                 // M -> M
        else if (lane == 22) hit = x < MSA_ANY && !(xb & 0x80) && xn == MSA_GAP;                 // M -> D
        else hit = false;
        if (hit) accv = __fadd_rn(accv, wi[k]);
      }
      float sum = 0.f;
#pragma unroll
      for (int a = 0; a < 20; ++a) sum = __fadd_rn(sum, __shfl_sync(0xffffffffu, accv, a));
      if (lane < 20)                     // NormalizeTo1(q->f[i], NAA, pb)
        F[(size_t)c * 20 + lane] = sum != 0.f ? __fmul_rn(accv, __double2float_rn(__ddiv_rn(1.0, (double)sum))) : pb[lane];
      const float mi = __shfl_sync(0xffffffffu, accv, 20), mm = __shfl_sync(0xffffffffu, accv, 21),
                  md = __shfl_sync(0xffffffffu, accv, 22);
      const float s3 = __fadd_rn(__fadd_rn(__fadd_rn(mm, mi), md), FLT_MIN);
      if (lane == 0) {
        TR[(size_t)c * 7 + 0] = flog2_dev(__fdiv_rn(mm, s3));
        TR[(size_t)c * 7 + 1] = flog2_dev(__fdiv_rn(mi, s3));
        TR[(size_t)c * 7 + 2] = flog2_dev(__fdiv_rn(md, s3));
        NEFF[c] = neff_run;
      }
    }
  }
}

// ---- Neff_HMM, insert and delete states, end states (:2640-2683, :2957-3382) -----------------------------------------
// Block per alignment.  The I and D states always use the global weights (the reference's "if (1)" branches).
__device__ __forceinline__ float msa_neff_from_w(float Nlim, float scale, float w) {
  // Nlim - (Nlim - 1.0) * fpow2(scale * w): float - double * float
  return __double2float_rn(__dsub_rn((double)Nlim, __dmul_rn(__dsub_rn((double)Nlim, 1.0), (double)fpow2_dev(__fmul_rn(scale, w)))));
}

__global__ void __launch_bounds__(256)
k_msa_finish(MsaArrays A, const float* __restrict__ pb, int use_global_weights, const float* __restrict__ lg2,
             const float* __restrict__ dif) {
  const int m = blockIdx.x;
  const MsaDesc d = A.desc[m];
  const int N = d.N, L = d.L, tid = threadIdx.x, T = blockDim.x;
  const uint8_t* X = A.X + d.x_off;
  const int8_t* in = A.keep + d.seq_off;
  const float* wg = A.wg + d.seq_off;
  float* F = A.f + d.col_off * 20;
  float* TR = A.tr + d.col_off * 7;
  float* NM = A.neff_m + d.col_off; float* NI = A.neff_i + d.col_off; float* ND = A.neff_d + d.col_off;
  const float* NEFF = A.neff_seg + d.col_off;
  const uint32_t* ins_off = A.ins_off + d.col_off;
  const int* ins_k = A.ins_k + d.ins_base; const uint16_t* ins_cnt = A.ins_cnt + d.ins_base;
  const int nf = A.n_filtered[m];
  const float NEG = -100000.0f;
  __shared__ float s_nhmm, s_nlim, s_scale;

  if (nf <= 1) {                           // "use first useful sequence" (:2111-2147)
    __shared__ int s_k;
    if (tid == 0) { int k = 0; for (; k < N; ++k) if (in[k]) break; s_k = k; if (k >= N) A.status[m] = 3; }
    __syncthreads();
    const int k = s_k;
    if (k >= N) return;
    const uint8_t* row = X + (size_t)k * d.stride;
    for (int i = tid; i <= L + 1; i += T) {
      const int x = (i == 0 || i == L + 1) ? MSA_ANY : msa_x(row, i);
      for (int a = 0; a < 20; ++a) F[(size_t)i * 20 + a] = x < MSA_ANY ? (a == x ? 1.0f : 0.0f) : pb[a];
      if (i <= L) {
        NM[i] = i == 0 ? 99.999f : 1.0f; NI[i] = i == 0 ? 99.999f : 0.0f; ND[i] = i == 0 ? 99.999f : 0.0f;
        float* t = TR + (size_t)i * 7;
        t[0] = 0.f; t[1] = NEG; t[2] = NEG; t[3] = (i == 0 || i == L) ? 0.f : NEG; t[4] = NEG; t[5] = i == 0 ? 0.f : NEG; t[6] = NEG;
      }
    }
    if (tid == 0) A.neff_hmm[m] = 1.0f;
    return;
  }

  // ---- Neff_M, Neff_HMM
  if (!use_global_weights) {
    if (tid == 0) {
      float s = 0.f;
      for (int i = 1; i <= L; ++i) s = __fadd_rn(s, NEFF[i]);
      s_nhmm = __fdiv_rn(s, (float)L);
    }
    for (int i = 1 + tid; i <= L; i += T) { const float v = NEFF[i]; NM[i] = v == 0.f ? 1.0f : v; }
  } else {
    // entropy of the weighted columns (:2642-2649); the columns are independent, the sum over them is ordered
    float* ent = NM;                       // Neff_M[i] is rewritten below
    for (int i = 1 + tid; i <= L; i += T) {
      float s = 0.f;
      for (int a = 0; a < 20; ++a) {
        const float v = F[(size_t)i * 20 + a];
        if ((double)v > 1E-10) s = __fsub_rn(s, __fmul_rn(v, fast_log2_dev(v, lg2, dif)));
      }
      ent[i] = fpow2_dev(s);
    }
    __syncthreads();
    if (tid == 0) {
      float s = 0.f;
      for (int i = 1; i <= L; ++i) s = __fadd_rn(s, ent[i]);
      s_nhmm = __fdiv_rn(s, (float)L);
    }
  }
  __syncthreads();
  if (tid == 0) {
    const float nh = s_nhmm;
    A.neff_hmm[m] = nh;
    const float Nlim = __double2float_rn(fmax(10.0, __dadd_rn((double)nh, 1.0)));
    s_nlim = Nlim;
    s_scale = flog2_dev(__double2float_rn(__ddiv_rn((double)__fsub_rn(Nlim, nh), __dsub_rn((double)Nlim, 1.0))));
  }
  __syncthreads();
  const float Nlim = s_nlim, scale = s_scale;
  const float w0 = __double2float_rn(__ddiv_rn(-1.0, (double)nf));

  for (int i = 1 + tid; i <= L; i += T) {
    float* t = TR + (size_t)i * 7;
    if (use_global_weights) {              // Neff_M from the weight of the rows with a residue or X (:2653-2663)
      float w = w0;
      for (int k = 0; k < N; ++k) if (in[k] && msa_x(X + (size_t)k * d.stride, i) <= MSA_ANY) w = __fadd_rn(w, wg[k]);
      NM[i] = w < 0.f ? 1.0f : msa_neff_from_w(Nlim, scale, w);
    }
    // insert state (:3103-3132)
    {
      float w = w0, i2m = 0.f, i2i = 0.f;
      int ncol = 0;
      for (uint32_t e = ins_off[i]; e < ins_off[i + 1]; ++e) {
        const int k = ins_k[e];
        if (!in[k]) continue;
        ++ncol;
        w = __fadd_rn(w, wg[k]);
        i2m = __fadd_rn(i2m, wg[k]);
        i2i = __fadd_rn(i2i, __fmul_rn(wg[k], (float)((int)ins_cnt[e] - 1)));
      }
      if (ncol > 0) {
        NI[i] = w < 0.f ? 1.0f : msa_neff_from_w(Nlim, scale, w);
        const float sum = __fadd_rn(i2m, i2i);
        t[3] = flog2_dev(__fdiv_rn(i2m, sum));
        t[4] = flog2_dev(__fdiv_rn(i2i, sum));
      } else { NI[i] = 0.f; t[3] = NEG; t[4] = NEG; }
    }
    // delete state (:3316-3352)
    {
      float w = w0, d2m = 0.f, d2d = 0.f;
      int ncol = 0;
      for (int k = 0; k < N; ++k) {
        if (!in[k]) continue;
        const uint8_t* row = X + (size_t)k * d.stride;
        if (msa_x(row, i) != MSA_GAP) continue;
        ++ncol;
        w = __fadd_rn(w, wg[k]);
        const int xn = msa_x(row, i + 1);
        if (xn == MSA_GAP) d2d = __fadd_rn(d2d, wg[k]);
        else if (xn <= MSA_ANY) d2m = __fadd_rn(d2m, wg[k]);
      }
      if (ncol > 0) {
        ND[i] = w < 0.f ? 1.0f : msa_neff_from_w(Nlim, scale, w);
        const float sum = __fadd_rn(d2m, d2d);
        t[5] = flog2_dev(__fdiv_rn(d2m, sum));
        t[6] = flog2_dev(__fdiv_rn(d2d, sum));
      } else { ND[i] = 0.f; t[5] = NEG; t[6] = NEG; }
    }
  }
  __syncthreads();
  if (tid == 0) {                          // begin / end states (:2625-2634, :3138-3143, :3372-3374)
    float* t0 = TR; float* tL = TR + (size_t)L * 7;
    t0[0] = 0.f; t0[1] = NEG; t0[2] = NEG; tL[0] = 0.f; tL[1] = NEG; tL[2] = NEG;
    t0[3] = 0.f; t0[4] = NEG; tL[3] = 0.f; tL[4] = NEG;
    t0[5] = 0.f; t0[6] = NEG;
    NM[0] = 99.999f; NI[0] = 99.999f; ND[0] = 99.999f;
  }
  if (tid < 20) { F[tid] = pb[tid]; F[(size_t)(L + 1) * 20 + tid] = pb[tid]; }
}

#ifndef HHG_EMUL
// ---- pseudocounts: the HHM loader's column step on the floats of k_msa_mstate / k_msa_finish ------------------------
// Thread per column j = 1..L of every alignment of the chunk; rec_off[m] = offsets of the ColRec output (L per record).
__global__ void __launch_bounds__(128)
k_msa_prepare(int m, const MsaDesc* __restrict__ desc, const long long* __restrict__ rec_off, MsaArrays A,
              const uint8_t* __restrict__ ss, const __grid_constant__ HhmPrepArgs P, const float* __restrict__ lg2,
              const float* __restrict__ diff, ColRec* __restrict__ out, long long total_cols,
              float* __restrict__ tr_full, const float* __restrict__ tau_host) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= total_cols) return;
  int lo = 0, hi = m - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (rec_off[mid] <= c) lo = mid; else hi = mid - 1; }
  const MsaDesc d = desc[lo];
  const int Lt = d.L, j = (int)(c - rec_off[lo]) + 1;
  const float* TR = A.tr + d.col_off * 7;
  const float* NM = A.neff_m + d.col_off; const float* NI = A.neff_i + d.col_off; const float* ND = A.neff_d + d.col_off;
  float tr_prev[7], tr_here[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) { tr_prev[k] = TR[(size_t)(j - 1) * 7 + k]; tr_here[k] = TR[(size_t)j * 7 + k]; }
  hhm_transitions_core(tr_prev, NM[j - 1], NI[j - 1], ND[j - 1], j - 1, Lt, P, lg2, diff);
  hhm_transitions_core(tr_here, NM[j], NI[j], ND[j], j, Lt, P, lg2, diff);
  if (tr_full) {
    float* dst = tr_full + (size_t)(rec_off[lo] + lo) * 7;
#pragma unroll
    for (int k = 0; k < 7; ++k) dst[(size_t)j * 7 + k] = tr_here[k];
    if (j == 1) {
#pragma unroll
      for (int k = 0; k < 7; ++k) dst[k] = tr_prev[k];
    }
  }
  float f[20];
#pragma unroll
  for (int a = 0; a < 20; ++a) f[a] = A.f[(d.col_off + j) * 20 + a];
  ColRec r;
  hhm_emissions(f, NM[j], P.pcm, P, tau_host != nullptr, tau_host ? tau_host[c] : 0.f, r.p);
  r.m2m = tr_prev[0]; r.m2d = tr_prev[2]; r.d2m = tr_prev[5]; r.d2d = tr_prev[6]; r.i2m = tr_prev[3];
  r.i2i = tr_here[4]; r.m2i = tr_here[1];
  r.ss = ss ? (uint32_t)ss[c] : 0u;
  out[c] = r;
}

#endif  // HHG_EMUL

}  // namespace hhg
