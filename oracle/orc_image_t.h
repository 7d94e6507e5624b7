/* orc_image_t.h -- the type-generic half of orc_image.c, included once per T (float, double) with
 *   T   the image scalar type
 *   S   the name suffix (_f, _d)
 *   EPS std::numeric_limits<T>::epsilon()
 * Each statement restates one of image_processing.cpp in T; -ffp-contract=off keeps every product and sum rounded
 * on its own. */
#define F_(name, s) name##s
#define F(name, s) F_(name, s)

static int F(cmp, S)(const void* a, const void* b) {
    const T x = *(const T*)a, y = *(const T*)b;
    return (x < y) ? -1 : (y < x) ? 1 : 0;
}

static T F(tmax, S)(T a, T b) { return (a < b) ? b : a; } /* std::max */
static T F(tmin, S)(T a, T b) { return (b < a) ? b : a; } /* std::min */

static T F(lum3, S)(T r, T g, T b) { return (r * (T)R_LUM + g * (T)G_LUM) + b * (T)B_LUM; }

/* AutoExposure::apply up to the clamp, shared by the LocalToneMapper (clamp = 0).  Returns 0 when the image is
 * left untouched (too few candidates, or not initialised). */
static int F(ae_stage, S)(orc_img_state* s, const orc_img_params* p, T* img, size_t npx, int rgb, int update_state,
                          int clamp) {
    const size_t nval = npx * (rgb ? 3 : 1);
    if (s->counter == 0 && update_state) {
        T* cand = (T*)malloc(sizeof(T) * (npx / AE_STRIDE + 1));
        size_t n = 0;
        for (size_t i = 0; i < npx; i += AE_STRIDE) {
            const T v = rgb ? F(lum3, S)(img[i * 3], img[i * 3 + 1], img[i * 3 + 2]) : img[i];
            if (v > 0) cand[n++] = v;
        }
        if (n < AE_MIN_NONZERO_POINTS) {
            free(cand);
            return 0;
        }
        qsort(cand, n, sizeof(T), F(cmp, S));
        const size_t k_lo = (size_t)((double)n * p->lo_percentile);
        const size_t k_hi = (size_t)((double)n * p->hi_percentile);
        s->lo = cand[k_lo];
        s->hi = cand[n - k_hi - 1];
        free(cand);
        if (!s->initialized) {
            s->initialized = 1;
            s->lo_state = s->lo;
            s->hi_state = s->hi;
        }
    }
    if (!s->initialized) return 0;
    if (update_state) {
        s->lo_state = p->damping * s->lo_state + (1.0 - p->damping) * s->lo;
        s->hi_state = p->damping * s->hi_state + (1.0 - p->damping) * s->hi;
    }
    const double scale = (1.0 - (p->lo_percentile + p->hi_percentile)) / (s->hi_state - s->lo_state);
    if (isinf(scale) || isnan(scale)) {
        const T m = (T)(0.5 / s->hi_state);
        for (size_t i = 0; i < nval; ++i) img[i] *= m;
    } else if (scale * (0.0 - s->lo_state) + p->lo_percentile <= 0.0) {
        const T a = (T)s->lo_state, m = (T)scale, c = (T)p->lo_percentile;
        for (size_t i = 0; i < nval; ++i) img[i] -= a;
        for (size_t i = 0; i < nval; ++i) img[i] *= m;
        for (size_t i = 0; i < nval; ++i) img[i] += c;
    } else {
        const T m = (T)((1.0 - p->hi_percentile) / s->hi_state);
        for (size_t i = 0; i < nval; ++i) img[i] *= m;
    }
    if (clamp)
        for (size_t i = 0; i < nval; ++i) img[i] = F(tmin, S)(F(tmax, S)(img[i], (T)0), (T)1);
    if (update_state) s->counter = (s->counter + 1) % p->update_every;
    return 1;
}

void F(orc_ae_update, S)(orc_img_state* s, const orc_img_params* p, T* img, size_t rows, size_t cols, int rgb,
                         int update_state) {
    F(ae_stage, S)(s, p, img, rows * cols, rgb, update_state, 1);
}

/* Eigen's FullPivLU(A).solve(rhs) for the h x 2 matrix A = [1, i]: complete pivoting (first strict maximum of |a|
 * in column-major order), the elimination, P, the unit-lower and upper triangular solves, Q.  x: 2 out. */
void F(orc_fullpivlu_fit, S)(const T* rhs, size_t h, T* x) {
    T* lu = (T*)malloc(sizeof(T) * 2 * h);
    T* c = (T*)malloc(sizeof(T) * h);
    T* col[2] = {lu, lu + h};
    for (size_t i = 0; i < h; ++i) {
        col[0][i] = 1;
        col[1][i] = (T)i;
    }
    const size_t size = h < 2 ? h : 2;
    size_t rowt[2] = {0, 1}, colt[2] = {0, 1}, nonzero = size;
    T maxpivot = 0;
    for (size_t k = 0; k < size; ++k) {
        size_t br = k, bc = k;
        T best = fabs(col[k][k]);
        for (size_t j = k; j < 2; ++j)
            for (size_t r = (j == k ? k + 1 : k); r < h; ++r)
                if (fabs(col[j][r]) > best) {
                    best = fabs(col[j][r]);
                    br = r;
                    bc = j;
                }
        if (best == 0) {
            nonzero = k;
            for (size_t q = k; q < size; ++q) rowt[q] = colt[q] = q;
            break;
        }
        if (best > maxpivot) maxpivot = best;
        rowt[k] = br;
        colt[k] = bc;
        if (br != k)
            for (int j = 0; j < 2; ++j) {
                const T t = col[j][k];
                col[j][k] = col[j][br];
                col[j][br] = t;
            }
        if (bc != k) {
            T* t = col[k];
            col[k] = col[bc];
            col[bc] = t;
        }
        for (size_t r = k + 1; r < h; ++r) col[k][r] = col[k][r] / col[k][k];
        if (k + 1 < size)
            for (size_t j = k + 1; j < 2; ++j)
                for (size_t r = k + 1; r < h; ++r) col[j][r] = col[j][r] - col[k][r] * col[j][k];
    }
    const T thr = maxpivot * ((T)EPS * (T)size);
    size_t rank = 0;
    for (size_t q = 0; q < nonzero; ++q) rank += fabs(col[q][q]) > thr;
    x[0] = x[1] = 0;
    if (rank > 0) {
        for (size_t i = 0; i < h; ++i) c[i] = rhs[i];
        for (size_t k = 0; k < size; ++k) {
            const T t = c[k];
            c[k] = c[rowt[k]];
            c[rowt[k]] = t;
        }
        if (size > 1) c[1] = c[1] - c[0] * col[0][1];
        if (rank > 1) {
            c[1] = c[1] / col[1][1];
            c[0] = c[0] - c[1] * col[1][0];
        }
        c[0] = c[0] / col[0][0];
        size_t q[2] = {0, 1};
        for (size_t k = 0; k < size; ++k) {
            const size_t t = colt[k], sv = q[k];
            q[k] = q[t];
            q[t] = sv;
        }
        for (size_t k = 0; k < rank; ++k) x[q[k]] = c[k];
    }
    free(lu);
    free(c);
}

/* compute_dark_count (image_processing.cpp:427-474); out: h values */
void F(orc_dark_count, S)(const T* img, size_t h, size_t w, T* out) {
    for (size_t i = 0; i < h; ++i) out[i] = 0;
    unsigned char* mask = (unsigned char*)calloc(w ? w : 1, 1);
    size_t n_cols = 0;
    for (size_t j = 0; j < w; ++j) {
        for (size_t i = 0; i < h && !mask[j]; ++i) mask[j] = img[i * w + j] != 0;
        n_cols += mask[j];
    }
    if (n_cols == 0) {
        free(mask);
        return;
    }
    T* tmp = (T*)malloc(sizeof(T) * n_cols);
    for (size_t i = 1; i < h; ++i) {
        size_t k = 0;
        for (size_t j = 0; j < w; ++j)
            if (mask[j]) tmp[k++] = img[i * w + j] - img[(i - 1) * w + j];
        qsort(tmp, n_cols, sizeof(T), F(cmp, S));
        out[i] = out[i - 1] + tmp[n_cols / 2];
    }
    T x[2];
    F(orc_fullpivlu_fit, S)(out, h, x);
    for (size_t i = 0; i < h; ++i) out[i] -= (T)1 * x[0] + (T)i * x[1];
    T m = out[0];
    for (size_t i = 1; i < h; ++i) m = F(tmin, S)(m, out[i]);
    for (size_t i = 0; i < h; ++i) out[i] -= m;
    free(tmp);
    free(mask);
}

/* BeamUniformityCorrector::apply; dark: the dark count, h doubles (its previous values when s->dc_rows == h) */
void F(orc_buc_update, S)(orc_img_state* s, double* dark, T* img, size_t h, size_t w, int update_state) {
    const int reset = s->dc_rows != (uint32_t)h;
    if (reset || (update_state && s->counter == 0)) {
        T* ndc = (T*)malloc(sizeof(T) * h);
        F(orc_dark_count, S)(img, h, w, ndc);
        for (size_t i = 0; i < h; ++i)
            dark[i] = reset ? (double)ndc[i] : dark[i] * BUC_DAMPING + (double)ndc[i] * (1.0 - BUC_DAMPING);
        s->dc_rows = (uint32_t)h;
        free(ndc);
    }
    s->counter = (s->counter + 1) % BUC_UPDATE_EVERY;
    for (size_t i = 0; i < h; ++i) {
        const T d = (T)dark[i];
        for (size_t j = 0; j < w; ++j) img[i * w + j] = F(tmax, S)(img[i * w + j] - d, (T)0);
    }
}

/* a NaN luminance goes to bin 0, as on the GPU; the reference's (int) cast of NaN is undefined and indexes out of
 * bounds on x86 */
static int F(clahe_bin, S)(T v) {
    const float f = (float)v * CLAHE_HIST_BINS;
    if (isnan(f)) return 0;
    const int b = (int)f;
    return b < CLAHE_HIST_BINS - 1 ? b : CLAHE_HIST_BINS - 1;
}

/* compute_clahe_luts (image_processing.cpp:86-133); luts: 8 * 8 * 1024 floats */
void F(orc_clahe_luts, S)(const T* lum, int h, int w, float* luts) {
    float hist[CLAHE_HIST_BINS];
    for (int ty = 0; ty < CLAHE_TILES; ++ty)
        for (int tx = 0; tx < CLAHE_TILES; ++tx) {
            const int y0 = ty * h / CLAHE_TILES, y1 = (ty + 1) * h / CLAHE_TILES;
            const int x0 = tx * w / CLAHE_TILES, x1 = (tx + 1) * w / CLAHE_TILES;
            const int tile_pixels = (y1 - y0) * (x1 - x0);
            for (int b = 0; b < CLAHE_HIST_BINS; ++b) hist[b] = 0.0f;
            for (int y = y0; y < y1; ++y)
                for (int x = x0; x < x1; ++x) hist[F(clahe_bin, S)(lum[(size_t)y * w + x])] += 1.0f;
            const float clip = 1.0f * (float)tile_pixels / (float)CLAHE_HIST_BINS;
            float excess = 0.0f;
            for (int b = 0; b < CLAHE_HIST_BINS; ++b)
                if (hist[b] > clip) {
                    excess += hist[b] - clip;
                    hist[b] = clip;
                }
            const float redistribute = excess / (float)CLAHE_HIST_BINS;
            float* lut = luts + (size_t)(ty * CLAHE_TILES + tx) * CLAHE_HIST_BINS;
            const float inv_pix = 1.0f / (float)tile_pixels;
            float cdf = 0.0f;
            for (int b = 0; b < CLAHE_HIST_BINS; ++b) {
                cdf += hist[b] + redistribute;
                lut[b] = orc_fminf_std(cdf * inv_pix, 1.0f);
            }
        }
}

/* LocalToneMapper::apply (image_processing.cpp:532-690) on an rgb image */
void F(orc_ltm_update, S)(orc_img_state* s, const orc_img_params* p, T* img, size_t rows, size_t cols,
                          int update_state) {
    const size_t npx = rows * cols;
    if (!F(ae_stage, S)(s, p, img, npx, 1, update_state, 0)) return;
    const T thresh = (T)0.8;
    if (s->hi_state < p->compress_dr_max_lum)
        for (size_t i = 0; i < npx * 3; i += 3) {
            const T lum = F(lum3, S)(img[i], img[i + 1], img[i + 2]);
            if (lum > thresh) {
                const T new_lum = thresh + orc_fast_log10((float)((double)(lum - thresh) + 1.0));
                const T scale = new_lum / lum;
                img[i] *= scale;
                img[i + 1] *= scale;
                img[i + 2] *= scale;
            }
        }
    for (size_t i = 0; i < npx * 3; ++i) {
        const T x = F(tmax, S)(img[i], (T)0);
        img[i] = x / ((T)1 + x);
    }
    T* lum_ae = (T*)malloc(sizeof(T) * (npx ? npx : 1));
    for (size_t i = 0; i < npx; ++i) lum_ae[i] = F(lum3, S)(img[3 * i], img[3 * i + 1], img[3 * i + 2]);
    const int h = (int)rows, w = (int)cols;
    float* luts = (float*)malloc(sizeof(float) * CLAHE_TILES * CLAHE_TILES * CLAHE_HIST_BINS);
    F(orc_clahe_luts, S)(lum_ae, h, w, luts);
    T color_factor = (T)0.75;
    const T ramp_start = (T)1.0, ramp_end = (T)0.5;
    if (s->hi_state < ramp_start)
        color_factor *= F(tmax, S)((T)0, (T)((s->hi_state - ramp_end) / (ramp_start - ramp_end)));
    const int plain = !p->color_correct || color_factor == (T)0;
    for (int y = 0; y < h; ++y) {
        const float ty_f = ((float)y + 0.5f) * CLAHE_TILES / h - 0.5f;
        int ty0 = (int)floorf(ty_f);
        ty0 = ty0 < 0 ? 0 : ty0 > CLAHE_TILES - 1 ? CLAHE_TILES - 1 : ty0;
        const int ty1 = ty0 + 1 < CLAHE_TILES - 1 ? ty0 + 1 : CLAHE_TILES - 1;
        const float fy = ty_f - (float)ty0;
        const float one_minus_fy = 1.0f - fy;
        for (int x = 0; x < w; ++x) {
            const float tx_f = ((float)x + 0.5f) * CLAHE_TILES / w - 0.5f;
            int tx0 = (int)floorf(tx_f);
            tx0 = tx0 < 0 ? 0 : tx0 > CLAHE_TILES - 1 ? CLAHE_TILES - 1 : tx0;
            const int tx1 = tx0 + 1 < CLAHE_TILES - 1 ? tx0 + 1 : CLAHE_TILES - 1;
            const float fx = tx_f - (float)tx0;
            const T lum_old = lum_ae[(size_t)y * w + x];
            const int bin = F(clahe_bin, S)(lum_old);
            const float* l0 = luts + (size_t)ty0 * CLAHE_TILES * CLAHE_HIST_BINS;
            const float* l1 = luts + (size_t)ty1 * CLAHE_TILES * CLAHE_HIST_BINS;
            const float mapped =
                one_minus_fy * ((1.0f - fx) * l0[tx0 * CLAHE_HIST_BINS + bin] + fx * l0[tx1 * CLAHE_HIST_BINS + bin]) +
                fy * ((1.0f - fx) * l1[tx0 * CLAHE_HIST_BINS + bin] + fx * l1[tx1 * CLAHE_HIST_BINS + bin]);
            const T lum_new = (T)mapped;
            const T scale = (lum_old > (T)1e-6) ? lum_new / lum_old : (T)1;
            T* c = img + 3 * ((size_t)y * w + x);
            for (int k = 0; k < 3; ++k) {
                if (plain) {
                    c[k] = F(tmin, S)(c[k] * scale, (T)1);
                } else {
                    T v = c[k] * scale;
                    v = -lum_new * color_factor + v * (1 + color_factor);
                    c[k] = F(tmax, S)((T)0, F(tmin, S)(v, (T)1));
                }
            }
        }
    }
    free(luts);
    free(lum_ae);
}

#undef F
#undef F_
