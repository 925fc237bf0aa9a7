/*
 * dsgd_host.c -- host-side data preparation for the SGD hot path (libdsgd_host.so, plain C, no CUDA).
 *
 * This is the data side of the boundary, the counterpart of utils/Dataset.scala (the reference builds its
 * `data: Array[(Vec, Int)]` on the JVM heap before any Slave exists).  It holds:
 *   - a deterministic generator of RCV1-shaped synthetic sparse rows (SURVEY.md 8d) -- there is no network
 *     and no RCV1 copy in this environment, so bench.py and the tests feed on this;
 *   - a parser for the RCV1 text format the reference reads (utils/Dataset.scala:19-45).
 * Nothing here touches weights or gradients; the arithmetic of the hot path is CUDA only.
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

/* ---- counter-based RNG: one independent stream per (seed, row) ------------------------------------- */
static inline uint64_t splitmix64(uint64_t *s) {
  uint64_t z = (*s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
typedef struct { uint64_t s; } rng_t;
static inline rng_t rng_for(uint64_t seed, uint64_t stream) {
  uint64_t s = seed * 0xD1342543DE82EF95ull + 0x2545F4914F6CDD1Dull;
  (void)splitmix64(&s);
  s ^= stream * 0x9E3779B97F4A7C15ull;
  (void)splitmix64(&s);
  rng_t r = {s};
  return r;
}
static inline double rng_u01(rng_t *r) { return (double)(splitmix64(&r->s) >> 11) * (1.0 / 9007199254740992.0); }
static inline double rng_normal(rng_t *r) { /* Box-Muller, one value per call */
  double u1 = rng_u01(r), u2 = rng_u01(r);
  if (u1 < 1e-300) u1 = 1e-300;
  return sqrt(-2.0 * log(u1)) * cos(6.283185307179586 * u2);
}

typedef struct {
  uint64_t seed;
  int64_t n_rows;
  int32_t dim;
  double mean_nnz;   /* 94.5: 0.2 % of 47 236 */
  double sigma;      /* lognormal shape of the row lengths */
  int32_t max_nnz;   /* 2000 */
  double zipf_s;     /* 1.1 */
  double zipf_q;     /* Zipf-Mandelbrot shift: p(rank) ~ 1/(rank + q)^s */
  double label_noise;/* 0.1 */
} dsgd_synth_params;

static int32_t row_len(const dsgd_synth_params *p, int64_t r, double mu) {
  rng_t g = rng_for(p->seed ^ 0xA5A5A5A5ull, (uint64_t)r);
  double l = floor(exp(mu + p->sigma * rng_normal(&g)) + 0.5);
  int32_t cap = p->max_nnz < p->dim ? p->max_nnz : p->dim;
  if (l < 1.0) l = 1.0;
  if (l > (double)cap) l = (double)cap;
  return (int32_t)l;
}

/* Pass 1: row_ptr[n_rows + 1].  Returns nnz (or -1). */
int64_t dsgd_synth_row_ptr(const dsgd_synth_params *p, int64_t *row_ptr) {
  if (!p || !row_ptr || p->n_rows <= 0 || p->dim <= 0) return -1;
  const double mu = log(p->mean_nnz) - 0.5 * p->sigma * p->sigma;
  row_ptr[0] = 0;
#pragma omp parallel for schedule(static)
  for (int64_t r = 0; r < p->n_rows; ++r) row_ptr[r + 1] = row_len(p, r, mu);
  for (int64_t r = 0; r < p->n_rows; ++r) row_ptr[r + 1] += row_ptr[r];
  return row_ptr[p->n_rows];
}

static int cmp_i32(const void *a, const void *b) { return (*(const int32_t *)a > *(const int32_t *)b) - (*(const int32_t *)a < *(const int32_t *)b); }

/* Pass 2: fill col (sorted ascending, unique per row), val (|N(0,1)|, row L2-normalised, fp32), label, and
 * the planted separator w_star[dim] (optional out). */
int dsgd_synth_fill(const dsgd_synth_params *p, const int64_t *row_ptr, int32_t *col, float *val, int8_t *label,
                    double *w_star_out) {
  if (!p || !row_ptr || !col || !val || !label) return -1;
  const int32_t D = p->dim;
  double *cdf = (double *)malloc(sizeof(double) * (size_t)D);
  int32_t *perm = (int32_t *)malloc(sizeof(int32_t) * (size_t)D);
  double *wstar = (double *)malloc(sizeof(double) * (size_t)D);
  if (!cdf || !perm || !wstar) { free(cdf); free(perm); free(wstar); return -1; }
  double acc = 0.0;
  for (int32_t k = 0; k < D; ++k) { acc += pow((double)k + p->zipf_q + 1.0, -p->zipf_s); cdf[k] = acc; }
  for (int32_t k = 0; k < D; ++k) cdf[k] /= acc;
  /* popularity rank -> column id: a fixed shuffle, so hot columns are scattered over the id space */
  rng_t g = rng_for(p->seed ^ 0x5EEDull, 1);
  for (int32_t k = 0; k < D; ++k) perm[k] = k;
  for (int32_t k = D - 1; k > 0; --k) {
    int32_t j = (int32_t)(rng_u01(&g) * (double)(k + 1));
    if (j > k) j = k;
    int32_t t = perm[k]; perm[k] = perm[j]; perm[j] = t;
  }
  g = rng_for(p->seed ^ 0x57A2ull, 2);
  for (int32_t k = 0; k < D; ++k) wstar[k] = rng_normal(&g);
  /* centre w* on its popularity-weighted mean so that x.w* is balanced around 0 although x > 0 */
  {
    double mu_pop = 0.0, prev = 0.0;
    for (int32_t k = 0; k < D; ++k) { mu_pop += (cdf[k] - prev) * wstar[perm[k]]; prev = cdf[k]; }
    for (int32_t k = 0; k < D; ++k) wstar[k] -= mu_pop;
  }
  if (w_star_out) memcpy(w_star_out, wstar, sizeof(double) * (size_t)D);

  int err = 0;
#pragma omp parallel
  {
    uint8_t *seen = (uint8_t *)calloc((size_t)D, 1);
    if (!seen) {
#pragma omp atomic write
      err = 1;
    }
#pragma omp for schedule(dynamic, 1024)
    for (int64_t r = 0; r < p->n_rows; ++r) {
      if (!seen) continue;
      const int64_t b = row_ptr[r];
      const int32_t len = (int32_t)(row_ptr[r + 1] - b);
      rng_t rg = rng_for(p->seed, (uint64_t)r);
      int32_t got = 0;
      while (got < len) {
        const double u = rng_u01(&rg);
        int32_t lo = 0, hi = D - 1; /* first k with cdf[k] > u */
        while (lo < hi) { int32_t mid = (lo + hi) >> 1; if (cdf[mid] > u) hi = mid; else lo = mid + 1; }
        const int32_t c = perm[lo];
        if (seen[c]) continue;
        seen[c] = 1;
        col[b + got++] = c;
      }
      for (int32_t k = 0; k < len; ++k) seen[col[b + k]] = 0;
      qsort(col + b, (size_t)len, sizeof(int32_t), cmp_i32);
      double nrm = 0.0;
      /* values: |N(0,1)|, then the row is L2-normalised (RCV1 rows are cosine-normalised tf-idf) */
      for (int32_t k = 0; k < len; ++k) { double v = fabs(rng_normal(&rg)) + 1e-3; val[b + k] = (float)v; nrm += v * v; }
      nrm = sqrt(nrm);
      double s = 0.0;
      for (int32_t k = 0; k < len; ++k) { val[b + k] = (float)((double)val[b + k] / nrm); s += (double)val[b + k] * wstar[col[b + k]]; }
      s += p->label_noise * rng_normal(&rg);
      label[r] = s >= 0.0 ? 1 : -1;
    }
    free(seen);
  }
  free(cdf); free(perm); free(wstar);
  return err ? -1 : 0;
}

/* ---- RCV1 text format (utils/Dataset.scala:19-45) ---------------------------------------------------
 * vectors file: "<rowId>  <k>:<v> <k>:<v> ..." (two separators after the id: parts.drop(2), Dataset.scala:27);
 * qrels file:   "<topic> <rowId> 1"; label = +1 iff topic == "CCAT" (Dataset.scala:43), and because the pairs
 * go through .toMap, the LAST line of a rowId decides (quirk Q10).
 * Keys in the file are the reference's 1-based feature ids; they are stored 0-based (key - 1).
 *
 * Two-call protocol: dsgd_rcv1_count sizes the arrays (nnz counts every pair, an upper bound), dsgd_rcv1_parse fills them;
 * its row_ptr[n_rows] is the number of distinct keys stored. */
int dsgd_rcv1_count(const char *vectors_path, int64_t *n_rows, int64_t *nnz) {
  FILE *f = fopen(vectors_path, "r");
  if (!f) return -1;
  int64_t rows = 0, nz = 0;
  int c, prev = '\n', any = 0;
  while ((c = fgetc(f)) != EOF) {
    if (c == ':') ++nz;
    if (c == '\n') { if (any) ++rows; any = 0; } else if (c != ' ' && c != '\r') any = 1;
    prev = c;
  }
  if (prev != '\n' && any) ++rows;
  fclose(f);
  *n_rows = rows; *nnz = nz;
  return 0;
}

int dsgd_rcv1_parse(const char *vectors_path, int32_t dim, int64_t n_rows, int64_t nnz, int64_t *row_ptr, int32_t *col,
                    float *val, int64_t *row_ids) {
  FILE *f = fopen(vectors_path, "r");
  if (!f) return -1;
  char *line = NULL; size_t cap = 0; ssize_t got;
  int64_t r = 0, k = 0;
  row_ptr[0] = 0;
  while ((got = getline(&line, &cap, f)) > 0) {
    char *s = line;
    while (*s == ' ') ++s;
    if (*s == '\n' || *s == '\r' || *s == 0) continue;
    if (r >= n_rows) { free(line); fclose(f); return -2; }
    char *end;
    row_ids[r] = strtoll(s, &end, 10);
    s = end;
    while (*s && *s != '\n' && *s != '\r') {
      while (*s == ' ') ++s;
      if (!*s || *s == '\n' || *s == '\r') break;
      long key = strtol(s, &end, 10);
      if (end == s || *end != ':') { free(line); fclose(f); return -3; }
      s = end + 1;
      double v = strtod(s, &end);
      if (end == s) { free(line); fclose(f); return -3; }
      s = end;
      if (key < 1 || key > dim) { free(line); fclose(f); return -4; }  /* Sparse.apply allows key == size (Q11) */
      /* the reference builds a Map per row (.toMap, Dataset.scala:26-32): a repeated key keeps its last value.  Keys come
       * sorted in RCV1 files, so a key above the row's last one is new without a search */
      int64_t at = k;
      if (k > row_ptr[r] && (int32_t)(key - 1) <= col[k - 1])
        for (int64_t q = row_ptr[r]; q < k; ++q)
          if (col[q] == (int32_t)(key - 1)) { at = q; break; }
      if (at == k) {
        if (k >= nnz) { free(line); fclose(f); return -2; }
        col[k] = (int32_t)(key - 1); ++k;
      }
      val[at] = (float)v;
    }
    row_ptr[++r] = k;
  }
  free(line);
  fclose(f);
  return (r == n_rows) ? 0 : -2;
}

/* labels[i] for row_ids[i]; rows without a qrels line get 0 (the reference would throw NoSuchElement). */
int dsgd_rcv1_labels(const char *qrels_path, const int64_t *row_ids, int64_t n_rows, int8_t *labels) {
  FILE *f = fopen(qrels_path, "r");
  if (!f) return -1;
  int64_t max_id = 0;
  for (int64_t i = 0; i < n_rows; ++i) if (row_ids[i] > max_id) max_id = row_ids[i];
  int8_t *by_id = (int8_t *)calloc((size_t)max_id + 1, 1);
  if (!by_id) { fclose(f); return -1; }
  char topic[64]; long long id; int one;
  while (fscanf(f, "%63s %lld %d", topic, &id, &one) == 3)
    if (id >= 0 && id <= max_id) by_id[id] = (strcmp(topic, "CCAT") == 0) ? 1 : -1;  /* last line wins (Q10) */
  fclose(f);
  for (int64_t i = 0; i < n_rows; ++i) labels[i] = by_id[row_ids[i]];
  free(by_id);
  return 0;
}

/* ---- every qrels line (multi-label topics) ----------------------------------------------------------------------------
 * The two-call protocol of dsgd_rcv1_count / dsgd_rcv1_parse over a qrels file ("<topic> <doc id> 1" per line):
 *   dsgd_rcv1_topics_count: *n_lines, the distinct topic names *n_names and the bytes they take with one NUL each.
 *   dsgd_rcv1_topics_parse: names_out receives the distinct names, NUL-terminated, in first-seen order; line i's topic is
 *   line_topic[i] (an index into that order) and its document line_doc[i].  The caller maps documents to rows, sorts the
 *   names and drops repeated (topic, doc) lines.
 * Both return 0, -1 (cannot open the file or allocate) or -2 (the file holds more than the sizes passed to parse). */
static int topics_scan(const char *path, int64_t cap_lines, int32_t cap_names, int64_t cap_bytes, char *names_out,
                       int32_t *line_topic, int64_t *line_doc, int64_t *n_lines, int32_t *n_names, int64_t *n_bytes) {
  FILE *f = fopen(path, "r");
  if (!f) return -1;
  int64_t lines = 0, bytes = 0, cap = 0;
  int32_t names = 0;
  int64_t *off = NULL;   /* name k starts at buf + off[k] */
  char *buf = NULL;
  int64_t buf_cap = 0;
  char topic[64]; long long id; int one, rc = 0;
  while (fscanf(f, "%63s %lld %d", topic, &id, &one) == 3) {
    int32_t k = 0;
    while (k < names && strcmp(buf + off[k], topic) != 0) ++k;
    if (k == names) {   /* a new name */
      const int64_t len = (int64_t)strlen(topic) + 1;
      if (names == cap) {
        cap = cap ? 2 * cap : 256;
        int64_t *o = (int64_t *)realloc(off, sizeof(int64_t) * (size_t)cap);
        if (!o) { rc = -1; break; }
        off = o;
      }
      if (bytes + len > buf_cap) {
        buf_cap = 2 * (bytes + len) + 4096;
        char *b = (char *)realloc(buf, (size_t)buf_cap);
        if (!b) { rc = -1; break; }
        buf = b;
      }
      memcpy(buf + bytes, topic, (size_t)len);
      off[names++] = bytes;
      bytes += len;
    }
    if (line_topic) {
      if (lines >= cap_lines) { rc = -2; break; }
      line_topic[lines] = k;
      line_doc[lines] = (int64_t)id;
    }
    ++lines;
  }
  fclose(f);
  if (rc == 0 && names_out) {
    if (names > cap_names || bytes > cap_bytes) rc = -2;
    else if (bytes) memcpy(names_out, buf, (size_t)bytes);
  }
  free(off);
  free(buf);
  if (rc == 0) { *n_lines = lines; *n_names = names; *n_bytes = bytes; }
  return rc;
}

int dsgd_rcv1_topics_count(const char *qrels_path, int64_t *n_lines, int32_t *n_names, int64_t *names_bytes) {
  return topics_scan(qrels_path, 0, 0, 0, NULL, NULL, NULL, n_lines, n_names, names_bytes);
}

int dsgd_rcv1_topics_parse(const char *qrels_path, int64_t n_lines, int32_t n_names, int64_t names_bytes, char *names_out,
                           int32_t *line_topic, int64_t *line_doc) {
  int64_t l, b; int32_t k;
  return topics_scan(qrels_path, n_lines, n_names, names_bytes, names_out, line_topic, line_doc, &l, &k, &b);
}

/* Writes rows in the reference's text format (for feeding the same data to a JVM run of the reference). */
int dsgd_rcv1_write(const char *vectors_path, const char *qrels_path, int64_t n_rows, const int64_t *row_ptr,
                    const int32_t *col, const float *val, const int8_t *label, int64_t first_id) {
  FILE *fv = fopen(vectors_path, "w");
  FILE *fq = fopen(qrels_path, "w");
  if (!fv || !fq) { if (fv) fclose(fv); if (fq) fclose(fq); return -1; }
  for (int64_t r = 0; r < n_rows; ++r) {
    fprintf(fv, "%lld ", (long long)(first_id + r));
    for (int64_t k = row_ptr[r]; k < row_ptr[r + 1]; ++k) fprintf(fv, " %d:%.9g", col[k] + 1, (double)val[k]);
    fputc('\n', fv);
    fprintf(fq, "%s %lld 1\n", label[r] > 0 ? "CCAT" : "GCAT", (long long)(first_id + r));
  }
  fclose(fv); fclose(fq);
  return 0;
}

/* ---- JVM-exact batch draws (SURVEY.md 8f N4) ------------------------------------------------------------
 * The reference seeds scala.util.Random (a wrapper of java.util.Random) with 0 (Main.scala:32) and, in every sync
 * step, shuffles each worker's index range afresh and slices it (core/Master.scala:184-187).  These functions
 * reproduce that stream: java.util.Random's 48-bit LCG (seed scrambling, next(bits), nextInt(bound)) and
 * scala.util.Random.shuffle of Scala 2.12 (Fisher-Yates from the top: for n = len down to 2: swap(n - 1, nextInt(n))).
 * Pinned in tests on java.util.Random's well-known outputs; the shuffle order itself cannot be cross-checked here
 * (no JVM in this image). */
#define JR_MULT 0x5DEECE66DULL
#define JR_MASK ((1ULL << 48) - 1)

void dsgd_jrandom_seed(uint64_t *state, int64_t seed) { *state = ((uint64_t)seed ^ JR_MULT) & JR_MASK; }

static inline int32_t jr_next(uint64_t *state, int bits) {
  *state = (*state * JR_MULT + 0xBULL) & JR_MASK;
  return (int32_t)(*state >> (48 - bits));
}

/* bound <= 0: nextInt(); else nextInt(bound) */
int32_t dsgd_jrandom_next_int(uint64_t *state, int32_t bound) {
  if (bound <= 0) return jr_next(state, 32);
  int32_t r = jr_next(state, 31);
  const int32_t m = bound - 1;
  if ((bound & m) == 0) return (int32_t)(((int64_t)bound * (int64_t)r) >> 31);
  for (int32_t u = r; (int32_t)((uint32_t)u - (uint32_t)(r = u % bound) + (uint32_t)m) < 0; u = jr_next(state, 31)) {}
  return r;
}

void dsgd_scala_shuffle_i32(uint64_t *state, int32_t *buf, int64_t len) {
  for (int64_t n = len; n >= 2; --n) {
    const int32_t k = dsgd_jrandom_next_int(state, (int32_t)n);
    const int32_t tmp = buf[n - 1]; buf[n - 1] = buf[k]; buf[k] = tmp;
  }
}

/* One epoch of Master.fit's draws for `n_groups` contiguous groups of `group_size` rows (the last may be shorter),
 * n_rows in total: for batch = 0, B, 2B, ... < max group length: for each group: shuffle a fresh copy of its range, take
 * [batch, batch + B).  out[(step * n_groups + k) * B + i] = row id or -1 where the slice is shorter.  Returns steps. */
int64_t dsgd_jvm_sync_epoch(uint64_t *state, int64_t n_rows, int64_t group_size, int32_t batch_size, int32_t *out,
                            int64_t out_capacity) {
  if (n_rows <= 0 || group_size <= 0 || batch_size <= 0) return -1;
  const int64_t n_groups = (n_rows + group_size - 1) / group_size;
  const int64_t max_len = group_size < n_rows ? group_size : n_rows;
  const int64_t steps = (max_len + batch_size - 1) / batch_size;
  if (steps * n_groups * batch_size > out_capacity) return -2;
  int32_t *buf = (int32_t *)malloc(sizeof(int32_t) * (size_t)max_len);
  if (!buf) return -3;
  for (int64_t s = 0; s < steps; ++s) {
    const int64_t batch = s * batch_size;
    for (int64_t k = 0; k < n_groups; ++k) {
      const int64_t lo = k * group_size, hi = (lo + group_size < n_rows) ? lo + group_size : n_rows, len = hi - lo;
      for (int64_t i = 0; i < len; ++i) buf[i] = (int32_t)(lo + i);
      dsgd_scala_shuffle_i32(state, buf, len);
      int32_t *dst = out + (s * n_groups + k) * batch_size;
      for (int64_t i = 0; i < batch_size; ++i) dst[i] = (batch + i < len) ? buf[batch + i] : -1;
    }
  }
  free(buf);
  return steps;
}

/* ---- batch draws of one epoch of Master.fit (core/Master.scala:179-187), fast form ----------------------------------
 * The reference shuffles every worker's whole index range afresh for every step and takes the slice
 * [batch, batch + B) of it (quirk Q5): a slice of a fresh uniform permutation is a uniform draw WITHOUT replacement of
 * min(B, len - batch) rows of the range.  This draws exactly that, for all steps and groups of one epoch, with Floyd's
 * subset sampling (O(B) per draw instead of the O(len) shuffle) from a counter-based generator keyed by
 * (seed, epoch, step, group): every rank draws the same batches, steps are independent (parallel), and the draw of
 * epoch e + 1 can be made while epoch e runs on the GPU.
 *   groups: n_groups ranges [g_start[k], g_start[k] + g_len[k]);  steps = ceil(max_k g_len[k] / B)
 *   out[(step * n_groups + k) * B + i] = row id, -1 where the slice is shorter than B; counts[step * n_groups + k] =
 *   rows drawn.  Returns the number of steps, or < 0. */
int64_t dsgd_draw_epoch(uint64_t seed, int64_t epoch, int32_t n_groups, const int64_t *g_start, const int64_t *g_len,
                        int32_t batch_size, int32_t *out, int32_t *counts, int64_t out_capacity) {
  if (n_groups <= 0 || batch_size <= 0 || !g_start || !g_len || !out || !counts) return -1;
  int64_t max_len = 0;
  for (int32_t k = 0; k < n_groups; ++k) {
    if (g_len[k] < 0 || g_start[k] < 0 || g_start[k] + g_len[k] > (int64_t)INT32_MAX) return -1;
    if (g_len[k] > max_len) max_len = g_len[k];
  }
  const int64_t steps = (max_len + batch_size - 1) / batch_size;
  if (steps * n_groups * (int64_t)batch_size > out_capacity) return -2;
  int hbits = 4;
  while ((1 << hbits) < 4 * batch_size) ++hbits;       /* open addressing, load <= 1/4 */
  const uint32_t hmask = (1u << hbits) - 1u;
  int failed = 0;
#pragma omp parallel
  {
    int64_t *table = (int64_t *)malloc(sizeof(int64_t) * ((size_t)hmask + 1));
    if (!table) {
#pragma omp atomic write
      failed = 1;
    } else {
#pragma omp for schedule(static)
      for (int64_t s = 0; s < steps; ++s) {
        for (int32_t k = 0; k < n_groups; ++k) {
          const int64_t len = g_len[k], batch = s * (int64_t)batch_size;
          int64_t m = len - batch;
          if (m > batch_size) m = batch_size;
          if (m < 0) m = 0;
          int32_t *dst = out + (s * n_groups + k) * (int64_t)batch_size;
          counts[s * n_groups + k] = (int32_t)m;
          for (int64_t i = m; i < batch_size; ++i) dst[i] = -1;
          if (m == 0) continue;
          rng_t g = rng_for(seed ^ 0x5EEDBA7C4ull ^ ((uint64_t)epoch << 20), (uint64_t)(s * n_groups + k));
          for (uint32_t i = 0; i <= hmask; ++i) table[i] = -1;
          /* Floyd: for j = len - m .. len - 1: t = uniform[0, j]; take t unless already taken, then take j */
          int64_t n_out = 0;
          for (int64_t j = len - m; j < len; ++j) {
            /* unbiased bounded draw: 64-bit multiply-shift with rejection (Lemire) */
            const uint64_t range = (uint64_t)j + 1;
            uint64_t x = splitmix64(&g.s);
            __uint128_t mm = (__uint128_t)x * range;
            uint64_t lo = (uint64_t)mm;
            if (lo < range) {
              const uint64_t thr = (0 - range) % range;
              while (lo < thr) { x = splitmix64(&g.s); mm = (__uint128_t)x * range; lo = (uint64_t)mm; }
            }
            int64_t t = (int64_t)(mm >> 64);
            uint32_t h = (uint32_t)((uint64_t)t * 0x9E3779B97F4A7C15ull >> 40) & hmask;
            int taken = 0;
            while (table[h] >= 0) { if (table[h] == t) { taken = 1; break; } h = (h + 1) & hmask; }
            if (taken) {
              t = j;
              h = (uint32_t)((uint64_t)t * 0x9E3779B97F4A7C15ull >> 40) & hmask;
              while (table[h] >= 0) h = (h + 1) & hmask;
            }
            table[h] = t;
            dst[n_out++] = (int32_t)(g_start[k] + t);
          }
        }
      }
      free(table);
    }
  }
  return failed ? -3 : steps;
}

/* ---- the async worker's without-replacement batch draw (dsgd_feistel.h), exported for the tests -------------------------- */
#include "dsgd_feistel.h"
uint32_t dsgd_feistel_pos(uint32_t x, uint64_t n, uint64_t key) {
  return dsgd_feistel(x, dsgd_feistel_half_bits(n), key, (uint32_t)n);
}

/* ---- the bootstrap calls' Poisson(1) draw (dsgd_bootstrap.h), exported for the tests ---------------------------------- */
#include "dsgd_bootstrap.h"
int dsgd_bootstrap_draw(uint64_t key, uint64_t b, uint64_t i) { return dsgd_boot_m(dsgd_boot_stream(key, b), i); }
