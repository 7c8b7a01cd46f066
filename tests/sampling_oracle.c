/* The top-k / top-p filter of the semantic and coarse stages (DESIGN.md §14), restated in plain C for the tests: upstream Bark's
 * filter (generate_text_semantic / generate_coarse) on the reference's float arithmetic, with libm's exp as the reference's softmax
 * (bark.cpp:184-199) calls it.  Written from the rule, independently of the library's kernel and of its host replay.
 *
 *   1. order: x descending, equal values (+0 == -0) by descending index (np.argsort(x, kind="stable")[::-1]); NaN above everything
 *   2. top-p: the reference's softmax of the sorted row (float max, e = (float) exp((double)(y - max)), sequential float sum, p = e / sum),
 *      then the sequential float cumulative sum c; sorted position j >= 1 is removed when c[j - 1] > top_p
 *   3. top-k: v = the min(k, n)-th largest value after step 2 (removed entries count as -inf); every entry < v is removed
 *
 * orc_filter_row sets the removed logits of row to -inf, writes mask[i] = 1 for the kept ones (mask may be NULL) and returns how many
 * were kept. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float x; int i; } entry;

static int before(const void * pa, const void * pb) {                 /* qsort: a comes first -> negative */
    const entry * a = (const entry *) pa, * b = (const entry *) pb;
    const int na = isnan(a->x), nb = isnan(b->x);
    if (na != nb) return na ? -1 : 1;
    if (!na && a->x != b->x) return a->x > b->x ? -1 : 1;
    return a->i > b->i ? -1 : 1;                                        /* equal values (or both NaN): the larger index first */
}

static int descending(const void * pa, const void * pb) {
    const float a = *(const float *) pa, b = *(const float *) pb;
    return a > b ? -1 : a < b ? 1 : 0;
}

int orc_filter_row(float * row, int n, int top_k, int use_top_p, float top_p, unsigned char * mask) {
    entry * s = (entry *) malloc((size_t) n * sizeof(entry));
    float * z = (float *) malloc((size_t) n * sizeof(float));
    unsigned char * removed = (unsigned char *) calloc((size_t) n, 1);
    for (int i = 0; i < n; i++) { s[i].x = row[i]; s[i].i = i; }
    qsort(s, (size_t) n, sizeof(entry), before);
    for (int j = 0; j < n; j++) z[j] = s[j].x;
    if (use_top_p) {
        float * p = (float *) malloc((size_t) n * sizeof(float));
        float maxl = -INFINITY, sum = 0.0f, c = 0.0f;
        for (int j = 0; j < n; j++) maxl = maxl < z[j] ? z[j] : maxl;  /* std::max(maxl, l) */
        for (int j = 0; j < n; j++) { p[j] = (float) exp((double) (z[j] - maxl)); sum += p[j]; }
        for (int j = 0; j < n; j++) p[j] /= sum;
        for (int j = 0; j < n; j++) {
            if (j > 0 && c > top_p) removed[j] = 1;                     /* c is c[j - 1] here */
            c += p[j];
        }
        for (int j = 0; j < n; j++) if (removed[j]) z[j] = -INFINITY;
        free(p);
    }
    if (top_k > 0) {
        float * t = (float *) malloc((size_t) n * sizeof(float));
        memcpy(t, z, (size_t) n * sizeof(float));
        qsort(t, (size_t) n, sizeof(float), descending);
        const float v = t[(top_k < n ? top_k : n) - 1];
        for (int j = 0; j < n; j++) if (z[j] < v) removed[j] = 1;
        free(t);
    }
    int kept = 0;
    for (int j = 0; j < n; j++) {
        const int i = s[j].i;
        if (removed[j]) row[i] = -INFINITY; else kept++;
        if (mask) mask[i] = !removed[j];
    }
    free(s); free(z); free(removed);
    return kept;
}
