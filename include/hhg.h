/* include/hhg.h -- C-ABI of the GPU-native (H100, sm_90a) HH-suite hot path (Viterbi HMM-HMM alignment +
 * cs219 ungapped prefilter).  Plain pointers and sizes only; no torch / C++ types.
 *
 * This is the boundary a reference maintainer binds to.  The reference (soedinglab/hh-suite) has no
 * FFI layer; the seam is two C++ member calls, and each entry point below names the reference
 * interface it replaces (paths relative to the reference tree):
 *
 *   ViterbiRunner::alignment            src/hhviterbirunner.h:55   -> hhg_viterbi_search
 *   Viterbi::Align                      src/hhviterbi.h:63         -> (inside hhg_viterbi_search)
 *   Viterbi::Backtrace                  src/hhviterbi.h:99         -> (inside hhg_viterbi_search)
 *   Viterbi::ExcludeAlignment           src/hhviterbi.h:112        -> hhg_viterbi_search(excl_*)
 *   HMMSimd::MapHMMVector               src/hhhmmsimd.h:35         -> hhg_db_create (device layout)
 *   HMMSimd::MapOneHMM                  src/hhhmmsimd.h:34         -> hhg_query_set
 *   ViterbiMatrix (backtrace bytes)     src/hhviterbimatrix.h:29   -> hhg_viterbi_debug_bt
 *   Prefilter::ungapped_sse_score       src/hhprefilter.h:108      -> hhg_prefilter_ungapped
 *   Prefilter::prefilter_db (stage 1)   src/hhprefilter.h:80       -> hhg_prefilter_ungapped
 *   Prefilter::swStripedByte            src/hhprefilter.h:112      -> hhg_prefilter_sw
 *   HHEntry::getTemplateHMM / HMM::Read src/hhdatabase.cpp:300, src/hhhmm.cpp:202 -> hhg_db_create_hhm
 *   PrepareTemplateHMM                  src/hhfunc.cpp:165         -> hhg_db_create_hhm + hhg_db_apply_null_model
 *   HHEntry::getTemplateHMM, survivors  src/hhdatabase.cpp:300, src/hhprefilter.cpp:561 -> hhg_dbstore_create + hhg_db_stage
 *   PosteriorDecoder::realign           src/hhposteriordecoder.h:67 -> hhg_mac_realign
 *   PosteriorDecoderRunner (hhblits_omp, one per query)               -> hhg_mac_realign_batch
 *
 * Error convention: every function returns 0 on success or a negative HHG_E* code;
 * hhg_last_error() returns a thread-local message.  (The reference logs and exit()s,
 * src/hhviterbimatrix.cpp:45; the host adapter maps a non-zero status to the same behaviour.)
 * Threading: one hhg_ctx per (host thread, GPU); calls on different contexts are independent
 * (hhblits_omp calls the path concurrently, src/hhblits_omp.cpp:119-138).
 *
 * Profile layout ("prepared profile" = what PrepareQueryHMM / PrepareTemplateHMM leave in HMM::p and
 * HMM::tr, src/hhfunc.cpp:121-202):
 *   p  : float[(L+2)*20]  p[i*20+a], i = 0..L+1                       (HMM::p,  src/hhhmm.h:153)
 *   tr : float[(L+1)*7]   tr[i*7+k], k = M2M,M2I,M2D,I2M,I2I,D2M,D2D  (HMM::tr, src/hhdecl.h:68), log2
 *   ss : uint8[L+2]       ss[i] = ss_pred[i]*11 + ss_conf[i]          (src/hhhmmsimd.cpp:133); may be NULL
 */
#ifndef HHG_H_
#define HHG_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HHG_OK 0
#define HHG_EINVAL (-1)   /* bad argument */
#define HHG_ECUDA (-2)    /* CUDA runtime error (message in hhg_last_error) */
#define HHG_ENOMEM (-3)   /* device or host allocation failed */
#define HHG_ENODEV (-4)   /* no usable sm_90 device: there is NO CPU fallback */

typedef struct hhg_ctx hhg_ctx;   /* one GPU + one stream + scratch */
typedef struct hhg_db hhg_db;     /* a device-resident shard of prepared target profiles */
typedef struct hhg_csdb hhg_csdb; /* a device-resident shard of cs219 column-state sequences */

/* Alignment parameters: the hot-path knobs of the reference's Parameters (src/hhdecl.cpp:82-127). */
typedef struct hhg_params {
  int local;        /* par.loc   (1)      : local (Smith-Waterman like) vs global            */
  float egq;        /* par.egq   (0)      : end-gap penalty query                             */
  float egt;        /* par.egt   (0)      : end-gap penalty template                          */
  float shift;      /* par.shift (-0.03)  : score offset per match-match cell                 */
  float ssw;        /* par.ssw   (0.11)   : secondary-structure weight                        */
  int use_ss;       /* 1 = PRED_PRED ss term during alignment (Viterbi::Align dispatch,       */
                    /*     src/hhviterbi.cpp:177; needs ss arrays on query and db + S33)      */
  float corr;       /* par.corr  (0.1)    : weight of the column-score correlation term       */
  int ssm;          /* par.ssm   (2)      : 2 = ss score is part of the alignment and is      */
                    /*     subtracted again from Hit.score (src/hhviterbi.cpp:236)             */
} hhg_params;

/* Per-target result: ViterbiResult (src/hhviterbi.h:21) + the scalar part of BacktraceResult (:34). */
typedef struct hhg_hit {
  float score;      /* raw Viterbi score (ViterbiResult::score)                               */
  int32_t i2, j2;   /* end of alignment  (ViterbiResult::i/j)                                 */
  int32_t i1, j1;   /* start of alignment (i_steps[nsteps], j_steps[nsteps])                  */
  int32_t nsteps;   /* BacktraceResult::count                                                 */
  int32_t matched_cols;
  int32_t path_off; /* offset of this target's state string in the `paths` buffer             */
  float hit_score;  /* Hit.score = score - score_ss + corr * sum_{d=1..4} sum_k S[k]S[k-d]       */
                    /*   (Viterbi::ScoreForBacktrace, src/hhviterbi.cpp:195-281)                 */
  float score_ss;   /* Hit.score_ss                                                            */
} hhg_hit;

const char* hhg_last_error(void);

/* device < 0: use the current CUDA device.  stream: a cudaStream_t cast to void* or NULL for a
 * private stream (bench.py passes torch's current stream so torch.cuda.Event brackets the work). */
int hhg_ctx_create(int device, void* stream, hhg_ctx** out);
int hhg_ctx_destroy(hhg_ctx* ctx);
int hhg_ctx_sync(hhg_ctx* ctx);
/* Number of kernels this context has launched so far (bench.py's gpu_launches). */
long long hhg_ctx_launch_count(hhg_ctx* ctx);

/* Build the device-resident target shard from n prepared profiles held in HOST memory.
 *   L[n]; p_off[n] = float offset of target k's p block inside `p`; tr_off[n] likewise inside `tr`;
 *   ss_off[n] = byte offset inside `ss` (ignored when ss == NULL).
 * Device layout: one 112-byte column record per target column j=1..L:
 *   {p[j][0..19], tr[j-1][M2M,M2D,D2M,D2D,I2M], tr[j][I2I,M2I], ss[j]}  (the operands of cell (.,j),
 *   src/hhviterbialgorithm.cpp:219-228,277). */
int hhg_db_create(hhg_ctx* ctx, int n, const int32_t* L, const int64_t* p_off, const int64_t* tr_off,
                  const int64_t* ss_off, const float* p, const float* tr, const uint8_t* ss,
                  hhg_db** out);
/* Same, but the emissions are the pseudocount-added probabilities BEFORE the null model is factored in
 * (what AddAminoAcidPseudocounts leaves in HMM::p, src/hhfunc.cpp:176-178) and pav[n*20] holds each
 * target's average amino-acid frequencies (HMM::pav).  The query-dependent step of PrepareTemplateHMM
 * -- HMM::IncludeNullModelInHMM, src/hhhmm.cpp:2059 -- then runs on the GPU for every new query:
 * hhg_db_apply_null_model(columnscore = par.columnscore: 0 pb, 1 (q.pav+t.pav)/2, 2 t.pav, 3 q.pav). */
int hhg_db_create_raw(hhg_ctx* ctx, int n, const int32_t* L, const int64_t* p_off, const int64_t* tr_off,
                      const int64_t* ss_off, const float* p, const float* tr, const uint8_t* ss,
                      const float* pav, hhg_db** out);
int hhg_db_apply_null_model(hhg_ctx* ctx, hhg_db* db, const float* q_pav, const float* pb, int columnscore);

/* ---- database load straight from HHM text records (SURVEY 8a rows a10 + a11; 8f-1) ------------------------
 * Replaces, once per database instead of once per (query, target):
 *   HHDatabaseEntry::getTemplateHMM -> HMM::Read          src/hhdatabase.cpp:300-336, src/hhhmm.cpp:202-691
 *   PrepareTemplateHMM up to CalculateAminoAcidBackground src/hhfunc.cpp:165-188
 *     (AddTransitionPseudocounts src/hhhmm.cpp:1722, PreparePseudocounts :1811, AddAminoAcidPseudocounts :1874,
 *      CalculateAminoAcidBackground :1854)
 * The text is tokenised on the host, all arithmetic (fpow2 of the emissions, both pseudocount steps, pav) runs in
 * CUDA kernels with the reference's operation types and order; the result is the same shard hhg_db_create_raw
 * builds from the reference's own prepared arrays, bit for bit.  Follow with hhg_db_apply_null_model per query.
 *
 * data/off/len: the `_hhm.ffdata` bytes and the (offset, length) columns of its `.ffindex` (lib/ffindex/src/ffindex.h:
 * ffindex_entry_t), n records.  Each record must be in HHM format with a NULL line (every record's own NULL line
 * is its background, as HMM::Read sets pb before using it, src/hhhmm.cpp:540-543,666-668).  R = the 20x20
 * pseudocount matrix of SetSubstitutionMatrix (R[a][b], src/hhfunc.cpp).  All pseudocount modes 0..3 of
 * HMM::AddAminoAcidPseudocounts; for mode 2 with pcc != 1 the admixture tau = f(powf(Neff/pcb, pcc)) is computed per
 * column on the host with the C library's powf (the call the reference makes), everything else on the device.
 * Errors (malformed record, LENG/column mismatch) name the record; the reference would warn and skip. */
typedef struct hhg_prep_params {
  float gapb, gapd, gape, gapf, gapg, gaph, gapi; /* Parameters::gap*, defaults 1, .15, 1, .6, .6, .6, .6       */
  int32_t pcm;                                    /* par.pc_hhm_nocontext_mode (2)                              */
  float pca, pcb, pcc;                            /* par.pc_hhm_nocontext_a/b/c (1.0, 1.5, 1.0)                 */
} hhg_prep_params;
int hhg_db_create_hhm(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                      const hhg_prep_params* pp, const float* R, hhg_db** out);
/* PrepareQueryHMM for an HHM-format query without context-specific pseudocounts (SURVEY 8a row a12, the par.nocontxt
 * branch of src/hhfunc.cpp:121-160: AddTransitionPseudocounts, PreparePseudocounts + AddAminoAcidPseudocounts,
 * CalculateAminoAcidBackground -- the same steps a template gets, run by the same kernels).  Fills the host arrays that
 * hhg_query_set / hhg_prefilter_build_profile take: p[(L+2)*20] (rows 0 and L+1 = pav like the reference), tr[(L+1)*7]
 * in HMM::tr order, ss[L+2] (may be NULL), pav[20], *neff = Neff_HMM.  L_cap = capacity of the caller's arrays in
 * columns.  The context-specific (CRF) pseudocounts of default hhblits stay in the reference's host code. */
int hhg_query_from_hhm(hhg_ctx* ctx, const char* rec, int64_t len, const hhg_prep_params* pp, const float* R,
                       int32_t L_cap, int32_t* L_out, float* p, float* tr, uint8_t* ss, float* pav, float* neff);
/* ---- A3M multiple alignments -> HMMs (SURVEY 8a row a10, 8f-1: the alignment branch of the database reader) ----------
 * Replaces, once per database instead of once per (query, target),
 *   HHEntry::getTemplateHMM, A3M branch          src/hhdatabase.cpp:441-449
 *     Alignment::Read                            src/hhalignment.cpp:181-544
 *     Alignment::Compress (par.M_template = 1)   :822-990
 *     Alignment::Filter -> Filter2               :1470-1473, :1598-1968
 *     Alignment::FrequenciesAndTransitions       :2047-2400  (global weights :2083-2108,
 *       Amino_acid_frequencies_and_transitions_from_M_state :2408-2683, Transitions_from_I_state :2957-3157,
 *       Transitions_from_D_state :3165-3382)
 * followed by the same PrepareTemplateHMM steps as hhg_db_create_hhm.  The text is scanned on the host (residue codes,
 * insert counts, the reference's own length sort); filter, sequence weights, frequencies, transitions and Neff run in
 * CUDA kernels with the reference's operation types and order.
 * One step of the reference is a hardware approximation: the position-specific weights use simdf32_rcp = RCPPS
 * (:2531), whose bits differ between CPU vendors.  The library samples the host's RCPPS for every possible integer
 * argument once and the kernel looks the values up: the HMM equals the one the reference computes ON THE SAME HOST,
 * bit for bit.
 * Not built: the -mark option. */
typedef struct hhg_msa_params {
  int32_t maxseq, maxcol, maxres;   /* par.maxseq 65535, par.maxcol 32765, par.maxres 20001 (src/hhdecl.cpp:10-14)       */
  int32_t M, mark;                  /* par.M / par.M_template: 1 A2M/A3M (match = upper case), 2 gap rule (Mgaps), 3 first  */
                                    /* sequence (-M a2m | <percent> | first); par.mark 0 is the only value built          */
  int32_t max_seqid, coverage, qid, Ndiff;   /* par.max_seqid_db 90, coverage_db 0, qid_db 0, Ndiff_db 100 (Filter)      */
  float qsc;                        /* par.qsc_db -20 (off); > -10 needs the substitution matrix S                      */
  int32_t wg;                       /* 0: position-specific weights (par.wg; what the realignment stage reads templates   */
                                    /* with), 1: global weights -- ViterbiRunner::alignment reads alignment templates    */
                                    /* with wg = 1 "for performance" (src/hhviterbirunner.cpp:143): use 1 for its shard   */
  int32_t Mgaps;                    /* par.Mgaps 50: with M = 2, columns with a larger weighted gap percentage are inserts */
} hhg_msa_params;
void hhg_msa_params_default(hhg_msa_params* mp);
/* Host only: number of match columns and of sequences of one A3M record, and whether it carries >ss_pred. */
int hhg_a3m_scan(const char* rec, int64_t len, const hhg_msa_params* mp, int32_t* L, int32_t* N_in, int32_t* has_ss);
/* Host only: the scanner hhg_db_create_a3m / hhg_msa_to_hmm run per record, exposed for inspection and CPU-side tests:
 * X[N_in*(L+2)] residue codes of columns 0..L+1 (0..19 amino acids, 20 ANY, 21 GAP, 22 ENDGAP; column 0 = ANY and
 * column L+1 = ENDGAP), I[N_in*(L+2)] insert counts after each column (may be NULL), keep[N_in] as Alignment::Read and
 * the "no residues" rule of Filter2 leave it, nres[N_in], ksort[N_in] the length order the filter walks (QSortInt). */
int hhg_a3m_parse(const char* rec, int64_t len, const hhg_msa_params* mp, int32_t L_cap, int32_t N_cap, int32_t* dims,
                  uint8_t* X, uint16_t* I, int8_t* keep, int32_t* nres, int32_t* ksort);
/* One alignment -> the HMM as Alignment::FrequenciesAndTransitions leaves it (no pseudocounts): what a QUERY alignment
 * becomes in hhblits (src/hhblits.cpp:1438-1453) and what the parity tests compare.
 *   S[400] substitution matrix in bits (only read by the qsc test, may be NULL), pb[20] background frequencies
 *   dims[6] = {L, N_in, N_filtered, kfirst, kss_pred, kss_conf};  keep[N_in] (may be NULL): 0 / 1 / 2 after the filter;
 *   wg[N_in] (may be NULL) global weights;  f[(L+2)*20];  tr[(L+1)*7] log2, HMM::tr order;
 *   neff[3*(L+1)] = Neff_M, Neff_I, Neff_D;  *neff_hmm;  ss[L+2] (may be NULL) = ss_pred*11 + ss_conf per column */
int hhg_msa_to_hmm(hhg_ctx* ctx, const char* rec, int64_t len, const hhg_msa_params* mp, const float* S, const float* pb,
                   int32_t L_cap, int32_t N_cap, int32_t* dims, int8_t* keep, float* wg, float* f, float* tr,
                   float* neff, float* neff_hmm, uint8_t* ss);
/* Compressed alignment databases (`<db>_ca3m.ffdata`, what UniClust ships): Alignment::ReadCompressed
 * (src/hhalignment.cpp:546-815; HHDatabaseEntry::getTemplateHMM, src/hhdatabase.cpp:303-326) -- a consensus row that is
 * shown but stays outside the profile, then one record per sequence {u32 entry in the sequence database, u16 start, u16
 * blocks, blocks x (u8 matches, s8 inserts (+) or gaps (-))} -- followed by the steps of the A3M path.  seqs = the
 * `<db>_sequence.ffdata` bytes and the offset / length columns of its `.ffindex` in index-file order (the reference
 * addresses entries by position, ffindex_get_entry_by_index); the header database only names rows and is not needed. */
typedef struct hhg_seqdb { int64_t n; const char* data; const int64_t* off; const int64_t* len; } hhg_seqdb;
int hhg_ca3m_scan(const char* rec, int64_t len, const hhg_seqdb* seqs, const hhg_msa_params* mp, int32_t* L, int32_t* N_in);
int hhg_ca3m_parse(const char* rec, int64_t len, const hhg_seqdb* seqs, const hhg_msa_params* mp, int32_t L_cap, int32_t N_cap,
                   int32_t* dims, uint8_t* X, uint16_t* I, int8_t* keep, int32_t* nres, int32_t* ksort);   /* host only */
int hhg_ca3m_to_hmm(hhg_ctx* ctx, const char* rec, int64_t len, const hhg_seqdb* seqs, const hhg_msa_params* mp,
                    const float* S, const float* pb, int32_t L_cap, int32_t N_cap, int32_t* dims, int8_t* keep, float* wg,
                    float* f, float* tr, float* neff, float* neff_hmm);
int hhg_db_create_ca3m(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len, const hhg_seqdb* seqs,
                       const hhg_msa_params* mp, const float* S, const float* pb, const hhg_prep_params* pp,
                       const float* R, hhg_db** out);
/* PrepareQueryHMM (nocontxt branch) for a query ALIGNMENT: the alignment -> HMM steps above with the caller's filter
 * parameters (hhblits: par.max_seqid / coverage / qid / qsc / Ndiff, src/hhblits.cpp:1438-1453), then the pseudocount
 * steps of hhg_query_from_hhm.  Outputs as hhg_query_from_hhm. */
int hhg_query_from_a3m(hhg_ctx* ctx, const char* rec, int64_t len, const hhg_msa_params* mp, const float* S, const float* pb,
                       const hhg_prep_params* pp, const float* R, int32_t L_cap, int32_t* L_out, float* p, float* tr,
                       uint8_t* ss, float* pav, float* neff);
/* The shard straight from the `_a3m.ffdata` records (uncompressed A3M text): same result object as hhg_db_create_hhm.
 * pb[20]: the background the reference holds when it reads the alignments (SetSubstitutionMatrix's, unless an HHM file
 * read earlier overwrote it -- HMM::Read does, src/hhhmm.cpp:543). */
int hhg_db_create_a3m(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                      const hhg_msa_params* mp, const float* S, const float* pb, const hhg_prep_params* pp,
                      const float* R, hhg_db** out);
/* ---- context-specific pseudocounts of the query (SURVEY 8a row a12, the DEFAULT branch of PrepareQueryHMM) ------------
 * Two engines, as in the reference: the CRF below (a `.crf` file, the default) and the context library after
 * hhg_crf_tail_host (any other file given to -contxt); both use the hhg_crf handle.
 * Replaces HMM::AddContextSpecificPseudocounts (src/hhhmm.cpp:1820-1849) = cs::Pseudocounts::AddTo(count profile, admix)
 * with the CRF engine (src/cs/crf_pseudocounts-inl.h:74-110, src/cs/pseudocounts-inl.h:41-73), used twice per query by
 * hhblits: for the query HMM (par.pc_hhm_context_engine: HHsearch admixture 0.9 / 4.0 / 1.0) and for the prefilter
 * profile (par.pc_prefilter_context_engine: CS-BLAST admixture 0.8 / 2.0).  hhg_crf_create parses the text of a `.crf`
 * file (HH-suite ships data/context_data.crf: 4000 states, window 13; the file itself is not part of this repository)
 * and keeps the weights on the device.  The context scores of all states at all columns are computed in a CUDA kernel
 * (ordered double sums); the log-sum-exp over the states calls exp() / log() of the host's C library, as the reference
 * does, so it runs on the library's host threads: every output equals the reference's, bit for bit.
 *   f[(L+2)*20] frequencies without pseudocounts (HMM::f, e.g. from hhg_msa_to_hmm), neff_m[L+1] (Neff_M),
 *   p[(L+2)*20] out: rows 1..L; with pav != NULL also CalculateAminoAcidBackground (pb, neff_hmm): pav and rows 0, L+1.
 * Limits: windows are odd and at most 63 columns (hhg_crf_create refuses others); 1 <= L <= 32767, the query limit of
 * hhg_query_set; crf must have been created on ctx's device.  Each is HHG_EINVAL before anything is allocated or launched.
 * Target-Neff admixture (par...target_neff >= 1) is not built (default 0). */
typedef struct hhg_crf hhg_crf;
typedef struct hhg_admix { int32_t kind; double pca, pcb, pcc; } hhg_admix;   /* kind 0 constant, 1 CS-BLAST, 2 HHsearch */
int hhg_crf_create(hhg_ctx* ctx, const char* text, int64_t len, hhg_crf** out);
int hhg_crf_destroy(hhg_crf* crf);
int hhg_crf_info(const hhg_crf* crf, int32_t* n_states, int32_t* window, double* pc);
int hhg_query_context_pseudocounts(hhg_ctx* ctx, const hhg_crf* crf, int32_t L, const float* f, const float* neff_m,
                                   float neff_hmm, const float* pb, const hhg_admix* admix, float* p, float* pav);
/* Host only (inspection / CPU-side tests): parse without a device; weights of one state (w[window*20], bias); the
 * per-column tail on caller-supplied context scores score[L*n_states] (overwritten with the state posteriors). */
int hhg_crf_parse_host(const char* text, int64_t len, hhg_crf** out);
int hhg_crf_state(const hhg_crf* crf, int32_t k, double* w, double* bias);
int hhg_crf_tail_host(const hhg_crf* crf, int32_t L, double* score, const float* f, const float* neff_m, const hhg_admix* admix,
                      float* p);
/* The generative engine: a context library (`-contxt` with any file that is not a `.crf`; HH-suite ships
 * data/context_data.lib: 4000 profiles, window 13).  InitializePseudocountsEngine (src/hhfunc.cpp:229-236) reads it with
 * cs::ContextLibrary, applies TransformToLog and builds cs::LibraryPseudocounts(lib, par.csw, par.csb) for both
 * engines; the handle this returns stands for that engine and goes to every hhg_crf_* call above and to
 * hhg_query_context_pseudocounts, with the same limits and the same bit-for-bit results.  The context scores are the
 * window-weighted emission scores of cs::Emission (src/cs/emission.h:87-103): window weights weight_center and
 * weight_center * weight_decay^d at distance d.  par.csw / par.csb are floats (src/hhdecl.h:260-261, defaults 1.6f and
 * 0.85f), so pass (double)1.6f and (double)0.85f to get what hhblits computes, not 1.6 and 0.85.  hhg_crf_state gives a
 * profile's log-probabilities in w and its log prior in bias; hhg_crf_info's pc is its central column in linear space.
 * Texts the reference reads but this library refuses (HHG_EINVAL, naming the profile and, where relevant, the
 * column): even windows and windows over 63 columns, a profile LENG other than the library's, a profile whose row
 * count is not LENG or that numbers a row twice, a row with fewer than 20 values, a negative, infinite or NaN PRIOR, and
 * a value v whose probability 2^(-v/1000) is 0 or infinite in double -- '*' among them: the reference reads it as log 0,
 * and 0 * log 0 makes every column whose window holds a zero count NaN.  Non-finite window weights are refused too.
 * hhg_crf_create refuses the text of a context library, and this call the text of a CRF. */
int hhg_context_library_create(hhg_ctx* ctx, const char* text, int64_t len, double weight_center, double weight_decay,
                               hhg_crf** out);
int hhg_context_library_parse_host(const char* text, int64_t len, double weight_center, double weight_decay, hhg_crf** out);
/* Host only: LENG and whether the record carries an ss_pred sequence (no numbers are parsed). */
int hhg_hhm_scan(const char* rec, int64_t len, int32_t* L, int32_t* has_ss);
/* Host only: the tokeniser hhg_db_create_hhm runs per record, exposed for inspection and CPU-side tests.
 *   f_mb[L*20]       emission integers of columns 1..L, file (alphabetical) amino-acid order, '*' = 99999
 *   trn_mb[(L+1)*10] rows 0..L: 7 transition integers (M2M,M2I,M2D,I2M,I2I,D2M,D2D) + Neff_M, Neff_I, Neff_D
 *   ss[L]            ss_pred*11 + ss_conf of columns 1..L;  null_mb[20] the NULL line */
int hhg_hhm_parse(const char* rec, int64_t len, int32_t L, int32_t* f_mb, int32_t* trn_mb, uint8_t* ss,
                  int32_t* null_mb, float* neff_hmm, int32_t* has_pc);
/* The resident binary database format = what the shard holds: 112-byte column records
 *   {float p[20]; float m2m, m2d, d2m, d2d, i2m, i2i, m2i; uint32 ss}   (p before the null model)
 * plus pav[n*20].  read_* copy them out (which: 0 = before the null model, 1 = after the last
 * hhg_db_apply_null_model), hhg_db_create_packed loads them back without any parsing. */
int hhg_db_read_cols(hhg_ctx* ctx, const hhg_db* db, int which, int64_t first, int64_t count, void* out);
int hhg_db_read_pav(hhg_ctx* ctx, const hhg_db* db, float* out);
int hhg_db_create_packed(hhg_ctx* ctx, int n, const int32_t* L, const void* cols_raw, int has_ss,
                         const float* pav, hhg_db** out);
/* Debug / parity: the 1025-entry lg2 table of fast_log2 the library uses for Hit.score. */
int hhg_debug_fastlog2_table(hhg_ctx* ctx, float* lg2_out);
int hhg_db_destroy(hhg_db* db);
int hhg_db_size(const hhg_db* db);          /* number of targets */
long long hhg_db_columns(const hhg_db* db); /* sum of target lengths */
int hhg_db_lengths(const hhg_db* db, int32_t* out /* [hhg_db_size] */);

/* ---- databases larger than device memory: a host-resident profile store and a staged shard ------------------------
 * The reference never holds the profile database in memory: Prefilter::prefilter_db hands the NAMES of its survivors on
 * (src/hhprefilter.cpp:561-590) and HHEntry::getTemplateHMM (src/hhdatabase.cpp:300-336) reads only those entries from
 * the mmap'd ffindex.  Here the cs219 shard (one byte per column) stays on the device, the 112-byte column records of
 * all profiles stay in page-locked, device-mapped HOST memory (hhg_dbstore), and a staged shard is a device cache over
 * them that holds each query's or query batch's survivors.
 *
 * hhg_dbstore_create: room for capacity_targets targets and capacity_cols columns (112 bytes each, plus 80 bytes of
 *   pav per target), allocated at once and page-locked; has_ss as in hhg_db_create_packed.
 * hhg_dbstore_append_packed: n more targets from host arrays in the format hhg_db_read_cols with which = 0 and
 *   hhg_db_read_pav write (lengths L[n], sum(L) records, pav[n*20]).
 * hhg_dbstore_append_db: all targets of a raw device shard (hhg_db_create_raw / _hhm / _a3m / _ca3m / _packed), so a
 *   database of any format is loaded chunk by chunk: create a shard of one chunk, append it, destroy it.
 * Both refuse, before anything is copied, what does not fit the capacity, a length outside [1, 32767], a shard whose
 * has_ss differs from the store's, and a shard that is not raw or is itself staged.  Targets are numbered in append
 * order: these are the GLOBAL ids.  A store is destroyed after the staged shards made over it. */
typedef struct hhg_dbstore hhg_dbstore;
int hhg_dbstore_create(hhg_ctx* ctx, int capacity_targets, long long capacity_cols, int has_ss, hhg_dbstore** out);
int hhg_dbstore_append_packed(hhg_dbstore* store, int n, const int32_t* L, const void* cols_raw, const float* pav);
int hhg_dbstore_append_db(hhg_ctx* ctx, hhg_dbstore* store, const hhg_db* db);
int hhg_dbstore_destroy(hhg_dbstore* store);
int hhg_dbstore_size(const hhg_dbstore* store);          /* number of targets appended */
long long hhg_dbstore_columns(const hhg_dbstore* store); /* sum of their lengths */
int hhg_dbstore_lengths(const hhg_dbstore* store, int32_t* out /* [hhg_dbstore_size] */);
/* hhg_db_create_staged: a raw shard of max_targets slots over an arena of max_cols columns, empty at first.  It is an
 *   hhg_db: hhg_viterbi_search(_batch), hhg_plan_create, hhg_db_apply_null_model, hhg_mac_realign(_batch) and the
 *   read_* calls take it with LOCAL ids = slots (hhg_db_size is max_targets, hhg_db_columns is max_cols, an empty
 *   slot has length 0 and is refused as a target).  The store must live on ctx's device.
 * hhg_db_stage: makes the n targets global_ids[] resident and writes their local ids to local_ids_out[n] (duplicates
 *   share a slot).  Resident targets keep their local id and are not copied.  Missing ones take free slots and free
 *   arena runs; when there is none, targets this call does not name are evicted, least recently staged first, until a
 *   run fits.  The records of all missing targets arrive in ONE kernel launch that reads the store through its
 *   device-mapped pointer, on the context's auxiliary stream; the context stream waits for it by event, the host does
 *   not.  After a call that copied or evicted anything the shard is as after hhg_db_create_packed (apply the null
 *   model again before a single-query search), earlier local ids of evicted targets are void, the context's search
 *   plan is rebuilt and an hhg_plan made before the call refuses to run; a call that found everything resident
 *   changes nothing.
 *   A call whose distinct targets need more slots or columns than the shard has is HHG_EINVAL (the message gives
 *   both numbers), as is an id outside the store; the shard is then unchanged.
 *   stats_out (may be NULL): what this call did.
 * hhg_db_staged_lookup: global id (-1 for an empty slot) and first arena column (the `first` of hhg_db_read_cols) of
 *   n local ids; either output may be NULL. */
typedef struct hhg_stage_stats {
  int64_t hits;      /* distinct targets that were already resident */
  int64_t copied;    /* distinct targets copied from the store       */
  int64_t bytes;     /* bytes written to the device for them         */
  int64_t evicted;   /* targets that lost their slot                 */
} hhg_stage_stats;
int hhg_db_create_staged(hhg_ctx* ctx, hhg_dbstore* store, int max_targets, long long max_cols, hhg_db** out);
int hhg_db_stage(hhg_ctx* ctx, hhg_db* db, int n, const int32_t* global_ids, int32_t* local_ids_out,
                 hhg_stage_stats* stats_out);
int hhg_db_staged_lookup(const hhg_db* db, int n, const int32_t* local_ids, int32_t* global_ids_out,
                         int64_t* first_col_out);

/* A staged shard whose source is the database's own ffindex records (HHM, A3M or compressed A3M) instead of a store:
 * nothing is parsed or held for a record until a stage call names it, so a database of tens of millions of alignments
 * needs no store and no load pass.
 * hhg_recsrc_create_hhm / _a3m / _ca3m: n records, record r = len[r] bytes at data + off[r].  The parameters mean what
 *   they mean for hhg_db_create_hhm / _a3m / _ca3m and are copied, as are off and len; data and the hhg_seqdb arrays
 *   are NOT copied or read here: the caller keeps them alive (typically an mmap of the ffdata) while the source lives.
 *   Creation cost does not depend on the records' size.  GLOBAL ids are record indices.  has_ss = 1 writes the ss
 *   bytes the resident loaders write (0 for a record without ss_pred); has_ss = 0 writes 0 everywhere, and the shard
 *   refuses ss searches like a resident shard without ss.
 * hhg_recsrc_destroy is refused while a staged shard made over the source lives.
 * hhg_db_create_staged_records: as hhg_db_create_staged over the source.  hhg_db_stage on it places targets exactly as
 *   over a store (same local ids, stats and evictions for the same id sequence), but the host first scans the request's
 *   missing records on its threads; a malformed record, a length outside [1, 32767] or an id outside the source is
 *   HHG_EINVAL naming the record, with the shard unchanged and nothing launched.  The targets to copy are then built in
 *   groups by the loaders' kernels and moved into their arena runs by k_stage_gather on the context stream.  The call
 *   blocks the host for the scan and the build.  A record that fails in the kernels (e.g. no sequence left after the
 *   filter) is HHG_EINVAL naming it and leaves the shard empty.
 * hhg_db_staged_neff: Neff_HMM of the targets in n slots of a record-sourced shard (hhg_hitlist_pvalues' t_neff);
 *   refused on a store-backed shard and on an empty slot. */
typedef struct hhg_recsrc hhg_recsrc;
int hhg_recsrc_create_hhm(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                          const hhg_prep_params* pp, const float* R, int has_ss, hhg_recsrc** out);
int hhg_recsrc_create_a3m(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                          const hhg_msa_params* mp, const float* S, const float* pb, const hhg_prep_params* pp,
                          const float* R, int has_ss, hhg_recsrc** out);
int hhg_recsrc_create_ca3m(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                           const hhg_seqdb* seqs, const hhg_msa_params* mp, const float* S, const float* pb,
                           const hhg_prep_params* pp, const float* R, int has_ss, hhg_recsrc** out);
int hhg_recsrc_destroy(hhg_recsrc* src);
int hhg_recsrc_size(const hhg_recsrc* src);
int hhg_db_create_staged_records(hhg_ctx* ctx, hhg_recsrc* src, int max_targets, long long max_cols, hhg_db** out);
int hhg_db_staged_neff(const hhg_db* db, int n, const int32_t* local_ids, float* neff_out);

/* Set the query (replaces HMMSimd::MapOneHMM).  S33: float[44*44] or NULL (needed iff use_ss). */
int hhg_query_set(hhg_ctx* ctx, int Lq, const float* p, const float* tr, const uint8_t* ss,
                  const float* S33, const hhg_params* par);

/* Switch the PRED_PRED ss term of the following searches on/off (hhg_params.use_ss) without re-sending the query: the
 * reference decides it per 8-target batch (consensus over the lanes, src/hhviterbirunner.cpp:14-26), so a runner
 * splits a mixed target list into the two groups.  Needs a query set with ss and S33. */
int hhg_set_use_ss(hhg_ctx* ctx, int use_ss);

/* -excl / -template_excl (par.exclstr, par.template_exclstr; ViterbiRunner::exclude_regions / exclude_template_regions,
 * src/hhviterbirunner.cpp:291-330): query rows q_lo[k]..q_hi[k] are switched off for every template column, template
 * columns t_lo[k]..t_hi[k] for every query row, in every following search of this context (1-based, inclusive; counts of
 * 0 clear the setting).  Works together with the excl_* path exclusions of hhg_viterbi_search(_batch), and applies to
 * hhg_mac_realign(_batch) as well (PosteriorDecoder::exclude_regions / exclude_template_regions,
 * src/hhposteriordecoder.cpp:100-152). */
int hhg_set_excluded_regions(hhg_ctx* ctx, int nq, const int32_t* q_lo, const int32_t* q_hi, int nt, const int32_t* t_lo,
                             const int32_t* t_hi);

/* Align the current query against `n` targets of `db` (ids == NULL: all targets in db order).
 *   hits[n]      : one record per requested target, in request order.
 *   paths        : caller buffer of `paths_cap` bytes (>= sum of nsteps; sum(Lq+Lt+2) always suffices)
 *                  receiving, per target and tightly packed at hits[k].path_off, nsteps state bytes
 *                  (ViterbiMatrix codes MM=2,GD=3,IM=4,DG=5,MI=6; byte 0 = step 1 = cell (i2,j2),
 *                  last byte = step nsteps, forced to MM like src/hhviterbi.cpp:147); may be NULL.
 *   excl_*       : optional cell-off input = previous alignments to exclude (alternative alignments,
 *                  src/hhviterbirunner.cpp:277-288): for request k, the path steps
 *                  excl_i/excl_j[excl_off[k] .. excl_off[k+1]) are masked with the +-40 cross of
 *                  Viterbi::ExcludeAlignment.  NULL = no cell-off (AlignWithOutCellOff variants).
 *                  Pass steps 1 .. nsteps-1 of every earlier alignment of that target: the reference's loop is
 *                  `for (step = 1; step < nsteps; step++)` (src/hhviterbi.cpp:61-77), the last step is NOT masked.
 *                  excl_off must start at 0 and be monotonic, 1 <= excl_i <= Lq, 1 <= excl_j <= Lt of the request's
 *                  target; anything else is refused with HHG_EINVAL.
 * All host buffers; copies in and out are part of the call. */
int hhg_viterbi_search(hhg_ctx* ctx, const hhg_db* db, int n, const int32_t* ids, hhg_hit* hits,
                       uint8_t* paths, size_t paths_cap, const int64_t* excl_off,
                       const int32_t* excl_i, const int32_t* excl_j);

/* ---- query-batch mode (SURVEY 8f-4) ---------------------------------------------------------------------------
 * hhblits_omp (src/hhblits_omp.cpp:119-160) runs one full HHblits per OpenMP thread, i.e. many independent queries
 * against the same mmap'd database at once.  Here a batch of queries shares ONE resident shard and ONE launch: the
 * work items (query, 32-target job, strip) of all queries feed the same persistent grid, which is what keeps the GPU
 * busy when each query only aligns the few thousand survivors of its prefilter (a single such request is latency
 * bound at ~100 GCUPS).
 *   hhg_query_set_batch : the queries (prepared like hhg_query_set; ss / S33 as there, ss may be NULL); q_pav[nq*20]
 *                         = HMM::pav of each query, needed when the shard is raw.  hhg_query_set == a batch of one.
 *   hhg_viterbi_search_batch : request k = (query req_query[k], target ids[k]); hits[k] / paths as in
 *                         hhg_viterbi_search (paths_cap >= sum(Lq_of_request + Lt + 2)).  Raw shard
 *                         (hhg_db_create_raw / _hhm / _packed): the query-dependent null model
 *                         (HMM::IncludeNullModelInHMM, columnscore / pb as in hhg_db_apply_null_model) is applied per
 *                         query while the plan's operand stream is built -- no per-query pass over the whole shard.
 *                         excl_*: as in hhg_viterbi_search, per request (the alternative alignments of
 *                         ViterbiRunner::alignment for every query of the batch in one call); steps are checked against
 *                         that request's query length and target length.  NULL = no path exclusions. */
int hhg_query_set_batch(hhg_ctx* ctx, int nq, const int32_t* Lq, const float* const* p, const float* const* tr,
                        const uint8_t* const* ss, const float* q_pav, const float* S33, const hhg_params* par);
int hhg_viterbi_search_batch(hhg_ctx* ctx, const hhg_db* db, int n, const int32_t* req_query, const int32_t* ids,
                             int columnscore, const float* pb, hhg_hit* hits, uint8_t* paths, size_t paths_cap,
                             const int64_t* excl_off, const int32_t* excl_i, const int32_t* excl_j);

/* Device-resident variant used for kernel-only timing: plan once, run many times, fetch at the end. */
typedef struct hhg_plan hhg_plan;
int hhg_plan_create(hhg_ctx* ctx, const hhg_db* db, int n, const int32_t* ids, hhg_plan** out);
int hhg_plan_destroy(hhg_plan* plan);
/* Enqueue forward pass + backtrace on the context stream; no host sync. */
int hhg_plan_run(hhg_ctx* ctx, hhg_plan* plan);
/* As hhg_plan_run, but brackets each forward-pass / backtrace launch with CUDA events on the context
 * stream and returns the summed device times in ms (synchronises). */
int hhg_plan_run_timed(hhg_ctx* ctx, hhg_plan* plan, float* ms_viterbi, float* ms_backtrace);
/* Copy results of the last run to the host (synchronises). paths may be NULL. */
int hhg_plan_fetch(hhg_ctx* ctx, hhg_plan* plan, hhg_hit* hits, uint8_t* paths, size_t paths_cap);
/* Device pointer to the plan's hit records (n x hhg_hit on the context's device), valid until the plan
 * is destroyed: lets the caller run the top-K selection / NCCL exchange without a host round trip. */
void* hhg_plan_hits_devptr(hhg_plan* plan);
/* sum over planned targets of Lq*Lt (the unit of the GCUPS metric) and padded cells actually computed */
double hhg_plan_cells(const hhg_plan* plan);
double hhg_plan_padded_cells(const hhg_plan* plan);
/* Algorithmic bytes of one run (SURVEY.md 8d): 112 B per target column + 1 B per cell + 32 B per hit */
double hhg_plan_algorithmic_bytes(const hhg_plan* plan);

/* ---- hit-list statistics (SURVEY 8a row a13; host side of the library, no GPU needed) ---------------------------
 * HitList::CalculatePvalues (src/hhhitlist.cpp:499-531): per hit the EVD parameters lamda, mu from the neural-network
 * regression over (query length, template length, query Neff, template Neff) (src/hhhitlist-inl.h:14-69), then
 * logPval / Pval (src/hhhit-inl.h:44-53) and Hit::CalcEvalScoreProbab (src/hhhit.h:134-194): Eval = Pval * N_searched,
 * score_aass (the list's sort key, more negative = better) and Probab.
 *   score / score_ss : Hit.score / Hit.score_ss (hhg_hit.hit_score / score_ss);  Lt, t_neff: template length and
 *   Neff_HMM;  hit_has_ss[k] != 0 iff the hit was scored with secondary structure (Hit.ssm1 || Hit.ssm2), may be NULL;
 *   loc, ssm, ssw = par.loc, par.ssm, par.ssw;  N_searched = number of database HMMs searched (global, all shards).
 * hhg_hitlist_hhblits_evalues (HitList::CalculateHHblitsEvalues, src/hhhitlist.cpp:465-494) overwrites Eval / logEval
 * with the prefilter-corrected composite E-value.  hhg_hitlist_order = HitList::SortList with Hit::operator<
 * (src/hhhit.h:116-126): ascending score_aass, then file name (strcmp; file may be NULL), then input order. */
typedef struct hhg_hit_stats {
  double Pval, logPval, Eval, logEval;
  float score_aass, Probab, lamda, mu;
} hhg_hit_stats;
int hhg_hitlist_pvalues(int n, const float* score, const float* score_ss, const int32_t* Lt, const float* t_neff,
                        const int32_t* hit_has_ss, int Lq, float q_neff, int N_searched, int loc, int ssm, float ssw,
                        hhg_hit_stats* out);
int hhg_hitlist_hhblits_evalues(int n, hhg_hit_stats* stats, const float* t_neff, float q_neff, int dbsize, float alphaa,
                                float alphab, float alphac, double prefilter_evalue_thresh);
int hhg_hitlist_order(int n, const hhg_hit_stats* stats, const char* const* file, int32_t* order);
/* ViterbiRunner::calculateEarlyStop (src/hhviterbirunner.cpp:213-247): sum over the hits of one chunk of 2000
 * database entries of 1/(1+Eval); hhblits stops aligning further chunks of the first alignment round when the sum is
 * below chunk_size * par.filter_thresh (:178-188).  score = Hit.score; prefilter = par.prefilter; dbsize = par.dbsize. */
float hhg_early_stop_sum(int n, const float* score, const int32_t* Lt, const float* t_neff, int Lq, float q_neff,
                         int prefilter, int dbsize, float alphaa, float alphab, float alphac,
                         double prefilter_evalue_thresh);

/* ---- multi-GPU: database sharded by target, hit lists merged over NCCL (SURVEY 8e) ------------------------------
 * The reference has no GPU or multi-device layer (its MPI front end distributes QUERIES, src/hhblits_mpi.cpp:135);
 * what must be kept is the result: every target aligned exactly once, one merged hit list ordered like a
 * single-process search (src/hhblits.cpp:890-905), global database size in the E-values.  One process (or host
 * thread) per GPU; each owns a shard (hhg_db) and a communicator.
 *   hhg_comm_unique_id : rank 0 obtains the 128-byte rendezvous id (ncclGetUniqueId) and hands it to the other
 *                        ranks by any means (argv, file, MPI, a shared variable between threads);
 *   hhg_comm_create    : collective over all ranks (ncclCommInitRank on the context's device); world == 1 needs
 *                        no NCCL at all.  NCCL is loaded at run time (libnccl.so.2; override with HHG_NCCL_LIB).
 *   hhg_plan_topk      : after hhg_plan_run / hhg_viterbi_search on every rank: selects this rank's K best hit
 *                        records on the GPU (radix select on a 64-bit key: score descending, GLOBAL target id
 *                        ascending), exchanges them with ONE ncclAllGather of K*56 bytes per rank and returns the
 *                        merged K best on every rank.  by_hit_score: 0 = raw Viterbi score, 1 = Hit.score.
 *                        Global id of request k = global_ids ? global_ids[k] : id_base + k  (host array of plan-n).
 *   hhg_plan_topk_paths: the state strings of the merged list (one ncclAllReduce of n_rec*width bytes; each row has
 *                        exactly one owner).  out[r*width ..] = path of recs[r], zero padded; width >= max nsteps. */
typedef struct hhg_comm hhg_comm;
typedef struct hhg_topk_rec {
  int32_t target;   /* global target id                          */
  int32_t owner;    /* rank whose shard holds it                 */
  hhg_hit hit;      /* the owner's hit record (path_off is local to the owner) */
  uint64_t key;     /* ordering key, ascending = better          */
} hhg_topk_rec;
int hhg_comm_unique_id(void* id128);
int hhg_comm_create(hhg_ctx* ctx, int rank, int world, const void* id128, hhg_comm** out);
int hhg_comm_destroy(hhg_comm* comm);
int hhg_comm_rank(const hhg_comm* comm);
int hhg_comm_world(const hhg_comm* comm);
int hhg_plan_topk(hhg_ctx* ctx, hhg_plan* plan, hhg_comm* comm, int K, int by_hit_score, int32_t id_base,
                  const int32_t* global_ids, hhg_topk_rec* out, int* n_out);
/* Same, ranked by a caller-supplied value per request, ASCENDING = better: key[k] = hhg_hit_stats.score_aass of
 * request k (hhg_hitlist_pvalues) gives exactly the reference's list order (Hit::operator<, src/hhhit.h:116-126). */
int hhg_plan_topk_by_key(hhg_ctx* ctx, hhg_plan* plan, hhg_comm* comm, int K, const float* key, int32_t id_base,
                         const int32_t* global_ids, hhg_topk_rec* out, int* n_out);
int hhg_plan_topk_paths(hhg_ctx* ctx, hhg_plan* plan, hhg_comm* comm, int n_rec, const hhg_topk_rec* recs, int width,
                        uint8_t* out);
/* The plan hhg_viterbi_search used last on this context (for hhg_plan_topk after a host-buffer search). */
hhg_plan* hhg_ctx_last_plan(hhg_ctx* ctx);

/* Debug / parity: raw backtrace bytes of request k of the last run of `plan` in the reference's
 * ViterbiMatrix cell format, row-major bt[i*(Lt+1)+j] (host buffer of (Lq+1)*(Lt+1) bytes). */
int hhg_plan_debug_bt(hhg_ctx* ctx, hhg_plan* plan, int k, uint8_t* bt);

/* ---- MAC realignment of reported hits (SURVEY 8f-3; the step after Viterbi) -------------------------------
 * Replaces PosteriorDecoder::realign (src/hhposteriordecoder.cpp:85-118) for a batch of hits of one query:
 * cell-off band around each hit's Viterbi path (maskViterbiAlignment :207-237) minus earlier MAC alignments of the
 * same template (excludeMACAlignment :242-258), Forward / Backward in double with the reference's row scaling
 * (src/hhforwardalgorithm.cpp, src/hhbackwardalgorithm.cpp), the MAC dynamic programme over posterior - mact
 * (src/hhmacalgorithm.cpp) and its backtrace (src/hhbacktracemac.cpp:112-210).  One warp per hit; every value is
 * computed with the reference's operation order and types, so posteriors, Pforward and paths are bit-identical.
 * The secondary-structure term: for predicted-vs-predicted structure (hit.ssm2 = 3) the reference's ScoreSS switch has
 * no such case (HMM::PRED_PRED = 4) and contributes exactly 0, so those hits are exact; not covered: DSSP-annotated
 * templates (hit.ssm2 = 1 or 2), self-alignment (hit.self).
 *
 * hhg_mac_query_set: q_p = HMM::p of the query, q_tr_lin = HMM::tr after Log2LinTransitionProbs(1.0)
 *   (src/hhposteriordecoderrunner.cpp:48); the boundary rows are reset here like initializeQueryHMMTransitions.
 * hhg_mac_realign, request r: target[r] = shard id (its records and transitions come from the resident shard; the
 *   linear transition probabilities are powf() of the shard's log2 values, computed by the host libm like the
 *   reference's HMM::Log2LinTransitionProbs);
 *   vit[5r..] = i1,i2,j1,j2,nsteps and vit_i/vit_j[vit_off[r] .. vit_off[r+1]) = Hit.i / Hit.j of steps 1..nsteps of
 *   the Viterbi alignment; excl_*: the (i,j) pairs of all earlier MAC alignments of this template (Hit.alt_i /
 *   alt_j, concatenated), or excl_off == NULL.
 * Outputs: hits[r]; the MAC path of request r sits at path_off..path_off+nsteps in out_i/out_j/out_states/out_post
 *   (index 0 unused, states 2 = MM, 4 = IM, 6 = MI; out_post = Hit.P_posterior).  path_cap >= sum(Lq + Lt + 2). */
typedef struct hhg_mac_params {
  int32_t local; /* par.loc   */
  float shift;   /* par.shift */
  float mact;    /* par.mact  */
} hhg_mac_params;
typedef struct hhg_mac_hit {
  int32_t i1, i2, j1, j2, nsteps, matched_cols;
  float sum_of_probs; /* Hit.sum_of_probs */
  int32_t flags;
  double pforward;    /* Hit.Pforward     */
  int64_t path_off;
} hhg_mac_hit;
/* Host only: HMM::Log2LinTransitionProbs(1.0), src/hhhmm.cpp:2305-2313, on n values. */
int hhg_log2lin(int64_t n, const float* in, float* out);
int hhg_mac_query_set(hhg_ctx* ctx, int Lq, const float* q_p, const float* q_tr_lin);
int hhg_mac_realign(hhg_ctx* ctx, const hhg_db* db, int n, const int32_t* target, const int32_t* vit,
                    const int64_t* vit_off, const int32_t* vit_i, const int32_t* vit_j, const int64_t* excl_off,
                    const int32_t* excl_i, const int32_t* excl_j, const hhg_mac_params* par, hhg_mac_hit* hits,
                    int32_t* out_i, int32_t* out_j, uint8_t* out_states, float* out_post, size_t path_cap);

/* Query batches (hhblits_omp runs one PosteriorDecoderRunner::executeComputation per query,
 * src/hhblits.cpp:973-1063 perform_realign): the hits of many queries realigned in one call.
 * hhg_mac_query_set_batch: nq queries as in hhg_mac_query_set; q_pav[nq*20] = HMM::pav of each query, needed when the
 *   shard is raw (may be NULL otherwise).  hhg_mac_query_set == a batch of one without q_pav.
 * hhg_mac_realign_batch, request r: query req_query[r] against target[r]; every other argument as in hhg_mac_realign,
 *   path_cap >= sum(Lq of the request's query + Lt + 2).  Raw shard (hhg_db_create_raw / _hhm / _packed): the null
 *   model of the request's query (HMM::IncludeNullModelInHMM, columnscore / pb as in hhg_viterbi_search_batch) is
 *   applied to a copy of the template's raw records, so the result does not depend on hhg_db_apply_null_model; a
 *   prepared shard is read as it is and columnscore / pb are ignored.  The requests are cut, in order, into memory waves
 *   whose scratch (about 6 bytes per cell) stays within the context's backtrace budget (HHG_MAX_BT_GB); the results
 *   do not depend on the cut.  Results are bit-identical to hhg_db_apply_null_model + hhg_mac_query_set +
 *   hhg_mac_realign per query. */
int hhg_mac_query_set_batch(hhg_ctx* ctx, int nq, const int32_t* Lq, const float* const* q_p,
                            const float* const* q_tr_lin, const float* q_pav);
int hhg_mac_realign_batch(hhg_ctx* ctx, const hhg_db* db, int n, const int32_t* req_query, const int32_t* target,
                          const int32_t* vit, const int64_t* vit_off, const int32_t* vit_i, const int32_t* vit_j,
                          const int64_t* excl_off, const int32_t* excl_i, const int32_t* excl_j,
                          int columnscore, const float* pb, const hhg_mac_params* par, hhg_mac_hit* hits,
                          int32_t* out_i, int32_t* out_j, uint8_t* out_states, float* out_post, size_t path_cap);
/* Debug / parity: the posterior matrix of request `request` of the last hhg_mac_realign(_batch), (Lq+1) x (Lt+1)
 * floats with the request's own Lq.  Refused after a call that ran in more than one memory wave. */
int hhg_mac_debug_posterior(hhg_ctx* ctx, int request, float* out);

/* ---- cs219 ungapped prefilter (stage 1 of Prefilter::prefilter_db, src/hhprefilter.cpp:466-482) */
int hhg_csdb_create(hhg_ctx* ctx, int n, const int32_t* L, const int64_t* off, const uint8_t* seq,
                    hhg_csdb** out);
int hhg_csdb_destroy(hhg_csdb* db);
/* The two set-up steps of the reference's Prefilter (SURVEY 8a row a18; ctor src/hhprefilter.cpp:28-47, init_prefilter
 * :314-335).  hhg_cs219_parse (host only): the text of the column-state library cs219.lib (the caller reads the file
 * that ships with HH-suite; cs::ContextLibrary / ContextProfile::Read) -> lib[k*20+a] linear probabilities, the
 * `lib219` argument of hhg_prefilter_build_profile; *n_states = 219.  hhg_csdb_create_ffindex: the shard straight
 * from <db>_cs219.ffdata and the (offset, length) columns of its .ffindex (length includes the NUL, like
 * ffindex_entry_t::length; sequence length = length - 1). */
int hhg_cs219_parse(const char* text, int64_t len, float* lib, int n_cap, int* n_states);
int hhg_csdb_create_ffindex(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                            hhg_csdb** out);
/* prof: uint8[220*Lq] linear query profile prof[k*Lq+pos] (the un-striped content of
 * Prefilter::stripe_query_profile, src/hhprefilter.cpp:356-424).  scores[n] receives the raw maximum
 * ungapped score per sequence (0..255), before the length correction of :477. */
int hhg_prefilter_ungapped(hhg_ctx* ctx, const hhg_csdb* db, int Lq, const uint8_t* prof, int offset,
                           int32_t* scores);
/* device-resident timing variant: scores stay on the device until fetched */
int hhg_prefilter_ungapped_run(hhg_ctx* ctx, const hhg_csdb* db, int Lq, const uint8_t* prof_host,
                               int offset, int upload_profile);
int hhg_prefilter_fetch(hhg_ctx* ctx, const hhg_csdb* db, int32_t* scores);
/* Stage-1 selection of Prefilter::prefilter_db on the device (src/hhprefilter.cpp:477-506), after
 * hhg_prefilter_ungapped_run: length correction score -= (int)(bit_factor*(flog2(Lq)+flog2(Lt))) (:477), then the
 * list sorted descending by (score, index) (:489-490) is kept "while count < min_hits or score > smax_thresh"
 * (:494-506).  Only the survivors leave the GPU (histogram + compaction; no N-element transfer or host sort).
 * ids/scores[cap] receive them in the reference's order, *n_out their number (HHG_EINVAL if it exceeds cap). */
int hhg_prefilter_select(hhg_ctx* ctx, const hhg_csdb* db, int Lq, int bit_factor, int smax_thresh,
                         int min_hits, int32_t* ids, int32_t* scores, int cap, int* n_out);

/* Host-side, once per query: the 220 x Lq byte profile of Prefilter::stripe_query_profile
 * (src/hhprefilter.cpp:356-424) in linear layout prof[k*Lq+pos].  q_p = HMM::p of the query
 * (float[(Lq+2)*20]), lib219 = 219x20 linear column-state probabilities of cs219.lib. */
int hhg_prefilter_build_profile(int Lq, const float* q_p, const float* q_pav, const float* lib219,
                                int score_offset, int bit_factor, uint8_t* prof);
/* Stage-1 length correction, src/hhprefilter.cpp:477. */
int hhg_prefilter_corrected_score(int raw, int Lq, int Lt, int bit_factor);
/* Stage-2 E-value, src/hhprefilter.cpp:529 (integer division of the score, fast fpow2). */
double hhg_prefilter_evalue(int score, long long num_dbs, int Lq, int Lt, int bit_factor);
/* Batch forms of the two formulas above (same arithmetic, element by element). */
int hhg_prefilter_corrected_scores(int n, const int32_t* raw, const int32_t* L, int Lq, int bit_factor,
                                   int32_t* out);
int hhg_prefilter_evalues(int n, const int32_t* score, const int32_t* L, long long num_dbs, int Lq,
                          int bit_factor, double* out);
/* Gapped stage 2 (Prefilter::swStripedByte, src/hhprefilter.cpp:70-212, AVX2 striping emulated lane for
 * lane) for n selected sequences of the shard (ids == NULL: the first n). gap_open is the reference's
 * gapOpen argument (= prefilter_gap_open + prefilter_gap_extend). scores[n]: host buffer. */
int hhg_prefilter_sw(hhg_ctx* ctx, const hhg_csdb* db, int n, const int32_t* ids, int Lq,
                     const uint8_t* prof, int gap_open, int gap_extend, int bias, int32_t* scores);

/* ---- cs219 prefilter for a batch of queries (hhblits_omp: one Prefilter::prefilter_db per query,
 * src/hhblits_omp.cpp).  Each call equals the single-query call made once per query, element by element.
 * prof[q]: uint8[220*Lq[q]] linear profile of query q, as hhg_prefilter_build_profile writes it.  All input is checked
 * before anything launches; bad input (nq < 1, a length < 1, a NULL profile, an offset outside 0..255, a request's
 * query or id out of range) returns HHG_EINVAL.
 *
 * hhg_prefilter_ungapped_batch_run: the ungapped stage of hhg_prefilter_ungapped for nq queries (nq <= 65535).  The
 * nq x n raw scores stay on the device in context scratch (hhg_csdb's single-query scores are not touched) until the
 * next batch run; hhg_prefilter_ungapped_batch_fetch copies them out, scores[q*n + k] = sequence k against query q.
 * Queries of up to 512 positions share one pass over the shard; a longer query takes one launch per 512 positions.
 * The nq x n score rows (raw and corrected, 8 bytes per query and sequence) must fit the context's memory budget
 * (HHG_MAX_BT_GB): a larger batch is refused with HHG_EINVAL, and hhg_prefilter_batch_max_queries says how many queries
 * fit (at least 1).  The edge bytes of long queries are cut into memory waves within what the score rows leave. */
int hhg_prefilter_batch_max_queries(hhg_ctx* ctx, const hhg_csdb* db);
int hhg_prefilter_ungapped_batch_run(hhg_ctx* ctx, const hhg_csdb* db, int nq, const int32_t* Lq,
                                     const uint8_t* const* prof, int offset);
int hhg_prefilter_ungapped_batch_fetch(hhg_ctx* ctx, const hhg_csdb* db, int32_t* scores);
/* hhg_prefilter_select_batch: hhg_prefilter_select for every query of the last batch run on this shard (nq must match
 * it), in two launches and two copies to the host whatever nq is.  Query q's survivors go to ids/scores[off[q] ..
 * off[q+1]) in the reference's order; off[nq+1] is filled even when the call fails because off[nq] exceeds cap
 * (HHG_EINVAL), so off[nq] is the capacity needed. */
int hhg_prefilter_select_batch(hhg_ctx* ctx, const hhg_csdb* db, int nq, const int32_t* Lq, int bit_factor,
                               int smax_thresh, int min_hits, int32_t* ids, int32_t* scores, int cap, int32_t* off);
/* hhg_prefilter_sw_batch: hhg_prefilter_sw for n requests in one launch; request r scores query req_query[r] against
 * sequence ids[r], scores[r] its result.  n = 0 is a no-op.  Same query length limit as hhg_prefilter_sw, checked for
 * the whole batch. */
int hhg_prefilter_sw_batch(hhg_ctx* ctx, const hhg_csdb* db, int nq, const int32_t* Lq, const uint8_t* const* prof,
                           int n, const int32_t* req_query, const int32_t* ids, int gap_open, int gap_extend, int bias,
                           int32_t* scores);

#ifdef __cplusplus
}
#endif
#endif /* HHG_H_ */
