// tdq_api.cu -- library-level entry points of the C ABI: errors, device query, mailbox, tableaus; and the host helpers
// every launcher shares (tdq_shape.cuh).
#include <stdarg.h>
#include <stdio.h>

#include "tdq_common.cuh"
#include "tdq_shape.cuh"

static thread_local char g_err[512] = "";

void tdq_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int tdq_sm_count() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
            sms = 132;
    }
    return sms;
}

void tdq_shape_from_tableau(const tdq_tableau *tab, TdqHostShape *h) {
    memset(h, 0, sizeof(*h));
    const int S = tab->n_stages;
    h->n_stages = S;
    h->fsal = tab->fsal;
    for (int i = 0; i < S; ++i) {
        int m = 0;
        for (int j = 0; j <= i; ++j)
            if (tab->beta[i][j] != 0.0) h->row_idx[i][m++] = j;
        h->row_nnz[i] = m;
    }
    int m = 0;
    for (int j = 0; j <= S; ++j)
        if (tab->c_sol[j] != 0.0) h->row_idx[S][m++] = j;
    h->row_nnz[S] = m;
    m = 0;
    for (int j = 0; j <= S; ++j)
        if (tab->c_err[j] != 0.0) h->err_idx[m++] = j;
    h->err_nnz = m;
    m = 0;
    for (int j = 0; j <= S; ++j)
        if (tab->c_mid[j] != 0.0) h->mid_idx[m++] = j;
    h->mid_nnz = m;
    h->valid = 1;
}

// ------------------------------------------------------------------------------------------------
// Butcher tableaus.  Coefficients are the published ones (Dormand & Prince 1980; Prince & Dormand
// 1981; Tsitouras 2011; Bogacki & Shampine 1989; Fehlberg 1969; Heun) written as the same rational
// expressions / decimal strings the reference evaluates in float64 (dopri5.py:5-30, dopri8.py:5-70,
// tsit5.py:6-75, bosh3.py:5-18, fehlberg2.py:4-18, adaptive_heun.py:5-21) so that both sides start
// from identical doubles.  Stored sparse: {row, column, value} triples; everything else is zero.
// ------------------------------------------------------------------------------------------------
namespace {

struct Entry { int i, j; double v; };
struct Vent { int j; double v; };

void fill(tdq_tableau *t, int S, int order, int fsal, const double *alpha, const Entry *b, int nb, const Vent *sol,
          int nsol, const Vent *err, int nerr, const Vent *mid, int nmid) {
    memset(t, 0, sizeof(*t));
    t->n_stages = S;
    t->order = order;
    t->fsal = fsal;
    for (int i = 0; i < S; ++i) t->alpha[i] = alpha[i];
    for (int e = 0; e < nb; ++e) t->beta[b[e].i][b[e].j] = b[e].v;
    for (int e = 0; e < nsol; ++e) t->c_sol[sol[e].j] = sol[e].v;
    for (int e = 0; e < nerr; ++e) t->c_err[err[e].j] = err[e].v;
    for (int e = 0; e < nmid; ++e) t->c_mid[mid[e].j] = mid[e].v;
}

void make_dopri5(tdq_tableau *t) {
    const double alpha[] = {1. / 5, 3. / 10, 4. / 5, 8. / 9, 1., 1.};
    const Entry b[] = {
        {0, 0, 1. / 5},
        {1, 0, 3. / 40}, {1, 1, 9. / 40},
        {2, 0, 44. / 45}, {2, 1, -56. / 15}, {2, 2, 32. / 9},
        {3, 0, 19372. / 6561}, {3, 1, -25360. / 2187}, {3, 2, 64448. / 6561}, {3, 3, -212. / 729},
        {4, 0, 9017. / 3168}, {4, 1, -355. / 33}, {4, 2, 46732. / 5247}, {4, 3, 49. / 176}, {4, 4, -5103. / 18656},
        {5, 0, 35. / 384}, {5, 2, 500. / 1113}, {5, 3, 125. / 192}, {5, 4, -2187. / 6784}, {5, 5, 11. / 84},
    };
    const Vent sol[] = {{0, 35. / 384}, {2, 500. / 1113}, {3, 125. / 192}, {4, -2187. / 6784}, {5, 11. / 84}};
    const Vent err[] = {
        {0, 35. / 384 - 1951. / 21600}, {2, 500. / 1113 - 22642. / 50085}, {3, 125. / 192 - 451. / 720},
        {4, -2187. / 6784 - -12231. / 42400}, {5, 11. / 84 - 649. / 6300}, {6, -1. / 60.},
    };
    const Vent mid[] = {
        {0, 6025192743. / 30085553152. / 2}, {2, 51252292925. / 65400821598. / 2},
        {3, -2691868925. / 45128329728. / 2}, {4, 187940372067. / 1594534317056. / 2},
        {5, -1776094331. / 19743644256. / 2}, {6, 11237099. / 235043384. / 2},
    };
    fill(t, 6, 5, 1, alpha, b, sizeof(b) / sizeof(b[0]), sol, 5, err, 6, mid, 6);
}

// Dense-output weights at the half step of DOPRI8 (dopri8.py:39-61): a quintic in h = 1/2 divided by 1/h.
double d8mid(double c5, double c4, double c3, double c2, double c1, double c0) {
    const double h = 1. / 2;
    const double h2 = h * h, h3 = h2 * h, h4 = h2 * h2, h5 = h4 * h;   // Python's h**k for k <= 5 is exact here
    return (c5 * h5 + c4 * h4 + c3 * h3 + c2 * h2 + c1 * h + c0) / (1 / h);
}

void make_dopri8(tdq_tableau *t) {
    const double alpha[] = {1. / 18, 1. / 12, 1. / 8, 5. / 16, 3. / 8, 59. / 400, 93. / 200,
                            5490023248. / 9719169821., 13. / 20, 1201146811. / 1299019798., 1, 1, 1};
    const Entry b[] = {
        {0, 0, 1. / 18},
        {1, 0, 1. / 48}, {1, 1, 1. / 16},
        {2, 0, 1. / 32}, {2, 2, 3. / 32},
        {3, 0, 5. / 16}, {3, 2, -75. / 64}, {3, 3, 75. / 64},
        {4, 0, 3. / 80}, {4, 3, 3. / 16}, {4, 4, 3. / 20},
        {5, 0, 29443841. / 614563906}, {5, 3, 77736538. / 692538347}, {5, 4, -28693883. / 1125000000},
        {5, 5, 23124283. / 1800000000},
        {6, 0, 16016141. / 946692911}, {6, 3, 61564180. / 158732637}, {6, 4, 22789713. / 633445777},
        {6, 5, 545815736. / 2771057229.}, {6, 6, -180193667. / 1043307555},
        {7, 0, 39632708. / 573591083}, {7, 3, -433636366. / 683701615}, {7, 4, -421739975. / 2616292301.},
        {7, 5, 100302831. / 723423059}, {7, 6, 790204164. / 839813087}, {7, 7, 800635310. / 3783071287.},
        {8, 0, 246121993. / 1340847787}, {8, 3, -37695042795. / 15268766246.}, {8, 4, -309121744. / 1061227803},
        {8, 5, -12992083. / 490766935}, {8, 6, 6005943493. / 2108947869}, {8, 7, 393006217. / 1396673457},
        {8, 8, 123872331. / 1001029789},
        {9, 0, -1028468189. / 846180014}, {9, 3, 8478235783. / 508512852}, {9, 4, 1311729495. / 1432422823},
        {9, 5, -10304129995. / 1701304382}, {9, 6, -48777925059. / 3047939560.}, {9, 7, 15336726248. / 1032824649},
        {9, 8, -45442868181. / 3398467696.}, {9, 9, 3065993473. / 597172653},
        {10, 0, 185892177. / 718116043}, {10, 3, -3185094517. / 667107341}, {10, 4, -477755414. / 1098053517},
        {10, 5, -703635378. / 230739211}, {10, 6, 5731566787. / 1027545527}, {10, 7, 5232866602. / 850066563},
        {10, 8, -4093664535. / 808688257}, {10, 9, 3962137247. / 1805957418}, {10, 10, 65686358. / 487910083},
        {11, 0, 403863854. / 491063109}, {11, 3, -5068492393. / 434740067}, {11, 4, -411421997. / 543043805},
        {11, 5, 652783627. / 914296604}, {11, 6, 11173962825. / 925320556}, {11, 7, -13158990841. / 6184727034.},
        {11, 8, 3936647629. / 1978049680}, {11, 9, -160528059. / 685178525}, {11, 10, 248638103. / 1413531060},
        {12, 0, 14005451. / 335480064}, {12, 5, -59238493. / 1068277825}, {12, 6, 181606767. / 758867731},
        {12, 7, 561292985. / 797845732}, {12, 8, -1041891430. / 1371343529}, {12, 9, 760417239. / 1151165299},
        {12, 10, 118820643. / 751138087}, {12, 11, -528747749. / 2220607170.}, {12, 12, 1. / 4},
    };
    const Vent sol[] = {
        {0, 14005451. / 335480064}, {5, -59238493. / 1068277825}, {6, 181606767. / 758867731},
        {7, 561292985. / 797845732}, {8, -1041891430. / 1371343529}, {9, 760417239. / 1151165299},
        {10, 118820643. / 751138087}, {11, -528747749. / 2220607170.}, {12, 1. / 4},
    };
    const Vent err[] = {
        {0, 14005451. / 335480064 - 13451932. / 455176623},
        {5, -59238493. / 1068277825 - -808719846. / 976000145},
        {6, 181606767. / 758867731 - 1757004468. / 5645159321.},
        {7, 561292985. / 797845732 - 656045339. / 265891186},
        {8, -1041891430. / 1371343529 - -3867574721. / 1518517206},
        {9, 760417239. / 1151165299 - 465885868. / 322736535},
        {10, 118820643. / 751138087 - 53011238. / 667516719},
        {11, -528747749. / 2220607170. - 2. / 45},
        {12, 1. / 4},
    };
    const Vent mid[] = {
        {0, d8mid(-6.3448349392860401388, 22.1396504998094068976, -30.0610568289666450593, 19.9990069333683970610,
                  -6.6910181737837595697, 1.0)},
        {5, d8mid(-39.6107919852202505218, 116.4422149550342161651, -121.4999627731334642623,
                  52.2273532792945524050, -7.6142658045872677172, 0.0)},
        {6, d8mid(20.3761213808791436958, -67.1451318825957197185, 83.1721004639847717481, -46.8919164181093621583,
                  10.7281392630428866124, 0.0)},
        {7, d8mid(7.3347098826795362023, -16.5672243527496524646, 9.5724507555993664382, -0.1890893225010595467,
                  0.5526637063753648783, 0.0)},
        {8, d8mid(32.8801774352459155182, -89.9916014847245016028, 87.8406057677205645007, -35.7075975946222072821,
                  4.2186562625665153803, 0.0)},
        {9, d8mid(-10.1588990526426760954, 22.6237489648532849093, -17.4152107770762969005, 6.2736448083240352160,
                  -0.6627209125361597559, 0.0)},
        {10, d8mid(-12.5401268098782561200, 32.2362340167355370113, -28.5903289514790976966,
                   10.3160881272450748458, -1.2636789001135462218, 0.0)},
        {11, d8mid(29.5553001484516038033, -82.1020315488359848644, 81.6630950584341412934, -34.7650769866611817349,
                   5.4106037898590422230, 0.0)},
        {12, d8mid(-41.7923486424390588923, 116.2662185791119533462, -114.9375291377009418170,
                   47.7457971078225540396, -7.0321379067945741781, 0.0)},
        {13, d8mid(20.3006925822100825485, -53.9020777466385396792, 50.2558364226176017553,
                   -19.0082099341608028453, 2.3537586759714983486, 0.0)},
    };
    fill(t, 13, 8, 1, alpha, b, sizeof(b) / sizeof(b[0]), sol, 9, err, 9, mid, 10);
}

#include "tdq_tableau_tsit5.inc"

void make_tsit5(tdq_tableau *t) {
    // Not FSAL by the reference's own test (rk_common.py:83: c_sol[-1] = 1/66 != 0), so y1 comes from the c_sol row.
    fill(t, 6, 5, 0, kTsit5Alpha, kTsit5Beta, (int)(sizeof(kTsit5Beta) / sizeof(kTsit5Beta[0])), kTsit5Sol,
         (int)(sizeof(kTsit5Sol) / sizeof(kTsit5Sol[0])), kTsit5Err, (int)(sizeof(kTsit5Err) / sizeof(kTsit5Err[0])),
         kTsit5Mid, (int)(sizeof(kTsit5Mid) / sizeof(kTsit5Mid[0])));
}

void make_bosh3(tdq_tableau *t) {
    const double alpha[] = {1. / 2, 3. / 4, 1.};
    const Entry b[] = {{0, 0, 1. / 2}, {1, 1, 3. / 4}, {2, 0, 2. / 9}, {2, 1, 1. / 3}, {2, 2, 4. / 9}};
    const Vent sol[] = {{0, 2. / 9}, {1, 1. / 3}, {2, 4. / 9}};
    const Vent err[] = {{0, 2. / 9 - 7. / 24}, {1, 1. / 3 - 1. / 4}, {2, 4. / 9 - 1. / 3}, {3, -1. / 8}};
    const Vent mid[] = {{1, 0.5}};
    fill(t, 3, 3, 1, alpha, b, 5, sol, 3, err, 4, mid, 1);
}

void make_fehlberg2(tdq_tableau *t) {
    const double alpha[] = {1. / 2, 1.0};
    const Entry b[] = {{0, 0, 1. / 2}, {1, 0, 1. / 256}, {1, 1, 255. / 256}};
    const Vent sol[] = {{0, 1. / 512}, {1, 255. / 256}, {2, 1. / 512}};
    const Vent err[] = {{0, -1. / 512}, {2, 1. / 512}};
    const Vent mid[] = {{1, 0.5}};
    fill(t, 2, 2, 0, alpha, b, 3, sol, 3, err, 2, mid, 1);
}

void make_adaptive_heun(tdq_tableau *t) {
    const double alpha[] = {1.};
    const Entry b[] = {{0, 0, 1.}};
    const Vent sol[] = {{0, 0.5}, {1, 0.5}};
    const Vent err[] = {{0, 0.5}, {1, -0.5}};
    const Vent mid[] = {{0, 0.5}};
    fill(t, 1, 2, 0, alpha, b, 1, sol, 2, err, 2, mid, 1);
}

}  // namespace

extern "C" {

int tdq_abi_version(void) { return TDQ_ABI_VERSION; }

size_t tdq_sizeof(int32_t which) {
    switch (which) {
        case 0: return sizeof(tdq_tableau);
        case 1: return sizeof(tdq_options);
        case 2: return sizeof(tdq_mailbox);
        case 3: return sizeof(TdqXBuf);
    }
    return 0;
}

const char *tdq_last_error(void) { return g_err; }

int tdq_device_sm_count(int *out) {
    TDQ_REQUIRE(out, "null argument");
    int dev = 0;
    TDQ_CHECK_CUDA(cudaGetDevice(&dev));
    TDQ_CHECK_CUDA(cudaDeviceGetAttribute(out, cudaDevAttrMultiProcessorCount, dev));
    return TDQ_OK;
}

int tdq_tableau_get(const char *name, tdq_tableau *out) {
    TDQ_REQUIRE(name && out, "null argument");
    if (!strcmp(name, "dopri5")) make_dopri5(out);
    else if (!strcmp(name, "dopri8")) make_dopri8(out);
    else if (!strcmp(name, "tsit5")) make_tsit5(out);
    else if (!strcmp(name, "bosh3")) make_bosh3(out);
    else if (!strcmp(name, "fehlberg2")) make_fehlberg2(out);
    else if (!strcmp(name, "adaptive_heun")) make_adaptive_heun(out);
    else {
        tdq_set_error("unknown tableau \"%s\"", name);
        return TDQ_ERR_INVALID;
    }
    return TDQ_OK;
}

int tdq_mailbox_create(tdq_mailbox **host_ptr, void **dev_ptr) {
    TDQ_REQUIRE(host_ptr && dev_ptr, "null argument");
    void *h = nullptr;
    TDQ_CHECK_CUDA(cudaHostAlloc(&h, sizeof(tdq_mailbox), cudaHostAllocMapped | cudaHostAllocPortable));
    memset(h, 0, sizeof(tdq_mailbox));
    void *d = nullptr;
    TDQ_CHECK_CUDA(cudaHostGetDevicePointer(&d, h, 0));
    *host_ptr = reinterpret_cast<tdq_mailbox *>(h);
    *dev_ptr = d;
    return TDQ_OK;
}

int tdq_mailbox_destroy(tdq_mailbox *host_ptr) {
    if (!host_ptr) return TDQ_OK;
    TDQ_CHECK_CUDA(cudaFreeHost(host_ptr));
    return TDQ_OK;
}

}  // extern "C"
