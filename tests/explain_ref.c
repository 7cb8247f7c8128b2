/* explain_ref.c -- CPU reference of rpk_explain (include/rpk.h), test infrastructure only.
 *
 * The GetGPUTypes filter loop (runpod_client.go:465-495, restated in oracle/rpk_oracle.c get_gpu_types) walked once
 * per pod with its predicate split apart: the cloud check and price > 0 decide whether the offer is offered at all, and
 * each of the four requirements is then tested on its own.  The rows are split over threads as rpk_oracle_select splits
 * them.  tests/explain_model.py builds this file into a temporary directory and loads it.  It lives beside the tests, not
 * in oracle/, because oracle/ is the fixed reference the existing suite measures against and is kept unchanged; the numpy
 * restatement in explain_model.py checks this loop independently. */
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>

#define CLOUD_SECURE 0
#define CLOUD_COMMUNITY 1

typedef struct {
    uint32_t n_feasible, n_unoffered, n_fail[4], n_only[4];
    int32_t nearest[4];
} explanation;

typedef struct {
    uint32_t G;
    const int32_t *mem_gb, *vcpu, *ram_gb; /* vcpu / ram_gb NULL = all 0 */
    const double *secure_price, *community_price;
    const uint8_t *flags;
    uint32_t p0, p1;
    const int32_t *req_mem_gb, *req_vcpu, *req_ram_gb; /* NULL = 0 */
    const double *max_price;                           /* NULL = 0.5 */
    const uint8_t *cloud;                              /* NULL = SECURE */
    explanation *out;
} explain_job;

static void explain_row(const explain_job *j, int32_t req_mem, int32_t req_vcpu, int32_t req_ram, double max_price,
                        int cloud_type, explanation *e) {
    double near_price[4] = {0, 0, 0, 0};
    *e = (explanation){0, 0, {0, 0, 0, 0}, {0, 0, 0, 0}, {-1, -1, -1, -1}};
    for (uint32_t g = 0; g < j->G; ++g) {
        double price = 0.0;
        int cloud_check = 0;
        if (cloud_type == CLOUD_SECURE) {
            price = j->secure_price[g];
            cloud_check = (j->flags[g] & 1) != 0;
        } else if (cloud_type == CLOUD_COMMUNITY) {
            price = j->community_price[g];
            cloud_check = (j->flags[g] & 2) != 0;
        }
        if (!(cloud_check && price > 0)) { ++e->n_unoffered; continue; }
        int32_t ov = j->vcpu ? j->vcpu[g] : 0;
        int32_t orm = j->ram_gb ? j->ram_gb[g] : 0;
        int fail[4];
        fail[0] = !(price < max_price);
        fail[1] = !(j->mem_gb[g] >= req_mem);
        fail[2] = !(ov >= req_vcpu);
        fail[3] = !(orm >= req_ram);
        int nf = fail[0] + fail[1] + fail[2] + fail[3];
        if (nf == 0) ++e->n_feasible;
        for (int r = 0; r < 4; ++r) {
            if (!fail[r]) continue;
            ++e->n_fail[r];
            if (nf != 1) continue;
            ++e->n_only[r];
            /* ascending g: a later offer replaces the nearest only at a strictly lower price */
            if (e->nearest[r] < 0 || price < near_price[r]) { e->nearest[r] = (int32_t)g; near_price[r] = price; }
        }
    }
}

static void *explain_range(void *arg) {
    const explain_job *j = (const explain_job *)arg;
    for (uint32_t p = j->p0; p < j->p1; ++p)
        explain_row(j, j->req_mem_gb[p], j->req_vcpu ? j->req_vcpu[p] : 0, j->req_ram_gb ? j->req_ram_gb[p] : 0,
                    j->max_price ? j->max_price[p] : 0.5, j->cloud ? j->cloud[p] : CLOUD_SECURE, &j->out[p]);
    return NULL;
}

int explain_ref(uint32_t G, const int32_t *mem_gb, const int32_t *vcpu, const int32_t *ram_gb, const double *secure_price,
                const double *community_price, const uint8_t *flags, uint32_t P, const int32_t *req_mem_gb,
                const int32_t *req_vcpu, const int32_t *req_ram_gb, const double *max_price, const uint8_t *cloud,
                explanation *out, int n_threads) {
    if (n_threads < 1) n_threads = 1;
    if ((uint32_t)n_threads > P && P > 0) n_threads = (int)P;
    explain_job *jobs = (explain_job *)calloc((size_t)n_threads, sizeof(explain_job));
    pthread_t *th = (pthread_t *)calloc((size_t)n_threads, sizeof(pthread_t));
    if (!jobs || !th) { free(jobs); free(th); return -1; }
    for (int i = 0; i < n_threads; ++i) {
        jobs[i] = (explain_job){G, mem_gb, vcpu, ram_gb, secure_price, community_price, flags,
                                (uint32_t)((uint64_t)P * (uint64_t)i / (uint64_t)n_threads),
                                (uint32_t)((uint64_t)P * (uint64_t)(i + 1) / (uint64_t)n_threads),
                                req_mem_gb, req_vcpu, req_ram_gb, max_price, cloud, out};
    }
    if (n_threads == 1) {
        explain_range(&jobs[0]);
    } else {
        for (int i = 0; i < n_threads; ++i) pthread_create(&th[i], NULL, explain_range, &jobs[i]);
        for (int i = 0; i < n_threads; ++i) pthread_join(th[i], NULL);
    }
    free(jobs); free(th);
    return 0;
}
