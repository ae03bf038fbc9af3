/*
 * dirt_oracle.c -- CPU ORACLE for the dirt rasterise / rasterise_grad hot path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product path
 * (dirt_b200/) never calls into oracle/.
 *
 * What it restates (paths relative to the reference checkout pmh47/dirt @ 95f5850):
 *   forward  : what OpenGL does for csrc/rasterise_egl.cpp:362-380 with the state set at
 *              :213-214,236,245 and the pass-through shaders csrc/shaders.cpp:16-43
 *              (clip -> NDC -> viewport, depth test LESS against 1.0, smooth = perspective-
 *              correct interpolation of vertex colours over the background); vertical
 *              orientation from csrc/rasterise_egl.cu:19-33,74-87.
 *   G-buffer : csrc/shaders.cpp:45-79 + csrc/rasterise_grad_egl.cpp:432-456
 *              (barycentrics, clip-space w = 1/gl_FragCoord.w, vertex indices; clear values
 *              (-1,-1,-1,+inf) / -1).
 *   backward : assemble_grads, csrc/rasterise_grad_egl.cu:93-236, line by line, including the
 *              per-channel-group behaviour of dirt/rasterise_ops.py:86-108,132-177 and the
 *              1-channel out-of-range channel reads of `at()` (:119-123).
 *
 * PARITY STATUS.  The forward arithmetic of the reference lives in the NVIDIA OpenGL driver
 * and raster hardware, which is not in the reference checkout and cannot run here (no TF, no
 * EGL/GL).  The only golden vector the reference holds for this path is
 * tests/square_test.py:11-17,54-57 (exact 128x128 equality), which this oracle is pinned
 * against (tests/test_oracle_golden.py).  Everything GL leaves implementation-defined is a
 * documented constant of THIS file (sub-pixel bits, tie rule, depth quantisation), and the
 * gradient values are pinned by no reference test: for those, "parity unpinned" -- parity
 * is defined as agreement with this restatement.
 *
 * ---------------------------------------------------------------------------------------
 * The visibility specification (bit-exact contract between this file and the CUDA kernels)
 * ---------------------------------------------------------------------------------------
 * All arithmetic below is IEEE-754, round-to-nearest-even, with NO fused contraction except
 * where fmaf() is written explicitly.  Build with -ffp-contract=off.
 *
 * Per face f = (i0,i1,i2) of image b, clip coordinates p_k = vertices[b,i_k] = (x,y,z,w):
 *  S1  any index outside [0,V) or any non-finite coordinate          -> face is culled.
 *  S2  "hard" faces: any w_k <= 0, or any snapped coordinate outside the guard band
 *      |X*256| <= 2^23 (32768 px).  Hard faces are rasterised per pixel in homogeneous
 *      form in double precision (H1-H3); all others are "normal" (S3-S7).
 *  S3  xn = x/w, yn = y/w (fp32 division);  X = (xn + 1) * (0.5*W);  Yd = (1 - yn) * (0.5*H)
 *      (Yd grows downwards: image row r spans Yd in [r, r+1], its centre is r + 0.5).
 *  S4  snap to 8 sub-pixel bits: xi = rint(X*256), yi = rint(Yd*256)  (int32).
 *  S5  area2 = cross(v1-v0, v2-v0) (int64).  0 -> culled.  <0 -> swap v1,v2 (coverage only).
 *      Edge k joins a = v(k+1), b = v(k+2):  A = ya-yb, B = xb-xa, C = -(A*xa + B*ya);
 *      E(P) = A*Px + B*Py + C > 0 inside.  Top-left rule in image space: an edge owns the
 *      points on it iff A > 0 or (A == 0 and B > 0).
 *      With pixel centres at (256c+128, 256r+128):
 *         q = floor((128*(A+B) + C - (topleft ? 0 : 1)) / 256)
 *         pixel (r,c) is covered  <=>  for all k: A_k*c + B_k*r + q_k >= 0     (int64)
 *  S6  interpolation planes come from the inverse of M = [x_k y_k w_k] (rows k) in double
 *      (inverse = cofactors * (1/det): one division, nine products):
 *      for a target t_k, (a,b,c) = M^-1 t solves a*x_k + b*y_k + c*w_k = t_k, and
 *      f(px,py) = a*px + b*py + c is the screen-space-affine function with f(ndc_k) = t_k/w_k.
 *      Converted to pixel indices (col,row):  gA = a*(2/W), gB = -b*(2/H),
 *      gC = a*(1/W - 1) + b*(1 - 1/H) + c.   det(M) == 0 or non-finite -> culled.
 *        depth   : t = z      -> Zwin = 0.5*f + 0.5 -> (zA,zB,zC) rounded to fp32, ABSOLUTE (col,row)
 *        q0, q1  : t = e0,e1  -> beta_k / w_k
 *        S       : t = (1,1,1)-> 1 / clip_w
 *      q0,q1,S planes are re-based to the reference pixel (cref,rref) = top-left pixel of the
 *      face's clamped bounding box and rounded to fp32.  A hard face with every w_k > 0 (it
 *      leaves the guard band; its bounding box is the frame) takes the frame pixel under its
 *      vertex of largest w instead: the first k with the largest w_k, (col,row) = (floor(X),
 *      floor(Yd)) of that vertex by S3 (fp32), clamped to [0,W-1] x [0,H-1].  There 1/clip_w is
 *      smallest; at (0,0) a small face far from the origin (frames past the guard band) would
 *      lose most of its precision.  A face with a vertex at w <= 0 keeps (0,0): its 1/clip_w
 *      plane crosses zero on screen, so no pixel anchors all of it better.
 *  S7  per pixel:  z = fmaf(zA, col, fmaf(zB, row, zC))           (fp32)
 *                  key = bits(fmaf(z, 2^23, 2^23)) - 0x4B000000   (uint32, wraps)
 *      fragment exists iff key < 2^23  (0 <= depth < 1.0: near/far clip and LESS against the
 *      cleared 1.0 in one test; key = rint(z*2^23), a 23-bit fixed-point depth).
 *      The visible face is the one with the smallest (key, face index).
 *  G   G-buffer at a covered pixel (fp32):  dc = col-cref, dr = row-rref,
 *      S  = fmaf(sA, dc, fmaf(sB, dr, sC));  clip_w = 1/S;
 *      q0 = fmaf(q0A, dc, fmaf(q0B, dr, q0C)), q1 likewise;
 *      bary = (q0*clip_w, q1*clip_w, 1 - q0*clip_w - q1*clip_w).
 *  H1  hard faces: the three planes q0,q1,q2 (t = e_k) and depth in double, absolute (col,row):
 *      v = gA*col + (gB*row + gC)   (double, no contraction).
 *  H2  covered iff for all k: q_k > 0 or (q_k == 0 and (gA_k > 0 or (gA_k == 0 and gB_k > 0))),
 *      and q0+q1+q2 > 0.
 *  H3  depth: z = (float)(Zwin plane in double); key as in S7.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

#define KEY_EMPTY 0x00800000u
#define GUARD_BAND 8388608.0f /* 2^23 sub-pixel units */

typedef struct {
    int kind; /* 0 culled, 1 normal, 2 hard */
    int v[3];
    int32_t A[3], B[3];
    int64_t q[3];
    int cmin, cmax, rmin, rmax; /* inclusive pixel bounding box (clamped to the frame) */
    float zA, zB, zC;
    float q0[3], q1[3], s[3]; /* (A,B,C) relative to (cref,rref) */
    int cref, rref;
    double hq[3][3]; /* hard: q_k planes (A,B,C), absolute */
    double hz[3];    /* hard: window depth plane, absolute */
} Tri;

typedef struct {
    int32_t A[3], B[3];
    int64_t q[3];
    float z[3];
    float q0[3], q1[3], s[3];
    int32_t cref, rref;
    int32_t kind;
    int32_t bbox[4];
} TriExport;

static inline uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

static inline uint32_t depth_key(float z)
{
    float zq = fmaf(z, 8388608.0f, 8388608.0f);
    return f2u(zq) - 0x4B000000u;
}

/* NDC plane (a,b,c) -> pixel-index plane (gA,gB,gC), all double, fixed operation order */
static void ndc_to_pixel_plane(double a, double b, double c, double two_over_W, double two_over_H,
                               double inv_W, double inv_H, double g[3])
{
    g[0] = a * two_over_W;
    g[1] = -(b * two_over_H);
    double t0 = a * (inv_W - 1.0);
    double t1 = b * (1.0 - inv_H);
    g[2] = (t0 + t1) + c;
}

static void setup_tri(const float* verts, const int32_t* face, int V, int H, int W, Tri* t)
{
    memset(t, 0, sizeof(*t));
    t->kind = 0;
    float p[3][4];
    for (int k = 0; k < 3; ++k) {
        int idx = face[k];
        if (idx < 0 || idx >= V) return;
        t->v[k] = idx;
        for (int j = 0; j < 4; ++j) {
            p[k][j] = verts[(size_t)idx * 4 + j];
            if (!isfinite(p[k][j])) return;
        }
    }
    int hard = 0;
    int n_behind = 0;
    for (int k = 0; k < 3; ++k)
        if (!(p[k][3] > 0.0f)) { hard = 1; ++n_behind; }
    if (n_behind == 3) return; /* entirely on the w <= 0 side: nothing can be visible */

    int32_t xi[3], yi[3];
    if (!hard) {
        const float halfW = 0.5f * (float)W, halfH = 0.5f * (float)H;
        for (int k = 0; k < 3; ++k) {
            float xn = p[k][0] / p[k][3];
            float yn = p[k][1] / p[k][3];
            float X = (xn + 1.0f) * halfW;
            float Y = (1.0f - yn) * halfH;
            float fx = X * 256.0f, fy = Y * 256.0f;
            if (!(fabsf(fx) <= GUARD_BAND) || !(fabsf(fy) <= GUARD_BAND)) { hard = 1; break; }
            xi[k] = (int32_t)lrintf(fx);
            yi[k] = (int32_t)lrintf(fy);
        }
    }

    /* S6: inverse of M in double */
    double x0 = p[0][0], y0 = p[0][1], w0 = p[0][3];
    double x1 = p[1][0], y1 = p[1][1], w1 = p[1][3];
    double x2 = p[2][0], y2 = p[2][1], w2 = p[2][3];
    double c00 = y1 * w2 - y2 * w1, c01 = y2 * w0 - y0 * w2, c02 = y0 * w1 - y1 * w0;
    double c10 = w1 * x2 - w2 * x1, c11 = w2 * x0 - w0 * x2, c12 = w0 * x1 - w1 * x0;
    double c20 = x1 * y2 - x2 * y1, c21 = x2 * y0 - x0 * y2, c22 = x0 * y1 - x1 * y0;
    double det = (x0 * c00 + y0 * c10) + w0 * c20;
    if (!(det != 0.0) || !isfinite(det)) return;
    const double rdet = 1.0 / det; /* one division, then products: part of the specification (S6) */
    double inv[3][3] = {{c00 * rdet, c01 * rdet, c02 * rdet},
                        {c10 * rdet, c11 * rdet, c12 * rdet},
                        {c20 * rdet, c21 * rdet, c22 * rdet}};
    const double two_over_W = 2.0 / (double)W, two_over_H = 2.0 / (double)H;
    const double inv_W = 1.0 / (double)W, inv_H = 1.0 / (double)H;
    double gq[3][3], gs[3], gz[3];
    for (int k = 0; k < 3; ++k)
        ndc_to_pixel_plane(inv[0][k], inv[1][k], inv[2][k], two_over_W, two_over_H, inv_W, inv_H, gq[k]);
    ndc_to_pixel_plane((inv[0][0] + inv[0][1]) + inv[0][2], (inv[1][0] + inv[1][1]) + inv[1][2],
                       (inv[2][0] + inv[2][1]) + inv[2][2], two_over_W, two_over_H, inv_W, inv_H, gs);
    {
        double z0 = p[0][2], z1 = p[1][2], z2 = p[2][2];
        double a = (inv[0][0] * z0 + inv[0][1] * z1) + inv[0][2] * z2;
        double b = (inv[1][0] * z0 + inv[1][1] * z1) + inv[1][2] * z2;
        double c = (inv[2][0] * z0 + inv[2][1] * z1) + inv[2][2] * z2;
        double g[3];
        ndc_to_pixel_plane(a, b, c, two_over_W, two_over_H, inv_W, inv_H, g);
        gz[0] = 0.5 * g[0];
        gz[1] = 0.5 * g[1];
        gz[2] = 0.5 * g[2] + 0.5;
    }
    for (int j = 0; j < 3; ++j)
        if (!isfinite(gz[j]) || !isfinite(gs[j]) || !isfinite(gq[0][j]) || !isfinite(gq[1][j]) || !isfinite(gq[2][j]))
            return;

    if (hard) {
        t->kind = 2;
        t->cmin = 0; t->cmax = W - 1; t->rmin = 0; t->rmax = H - 1;
        t->cref = 0; t->rref = 0;
        if (n_behind == 0) { /* past the guard band: the pixel under the first vertex of largest w */
            int kf = 0;
            if (p[1][3] > p[kf][3]) kf = 1;
            if (p[2][3] > p[kf][3]) kf = 2;
            const float X = floorf((p[kf][0] / p[kf][3] + 1.0f) * (0.5f * (float)W));
            const float Yd = floorf((1.0f - p[kf][1] / p[kf][3]) * (0.5f * (float)H));
            t->cref = !(X >= 0.0f) ? 0 : (X > (float)(W - 1) ? W - 1 : (int)X);
            t->rref = !(Yd >= 0.0f) ? 0 : (Yd > (float)(H - 1) ? H - 1 : (int)Yd);
        }
        for (int k = 0; k < 3; ++k)
            for (int j = 0; j < 3; ++j) t->hq[k][j] = gq[k][j];
        for (int j = 0; j < 3; ++j) t->hz[j] = gz[j];
    } else {
        int64_t ax = xi[0], ay = yi[0], bx = xi[1], by = yi[1], cx = xi[2], cy = yi[2];
        int64_t area2 = (bx - ax) * (cy - ay) - (cx - ax) * (by - ay);
        if (area2 == 0) return;
        int32_t px[3] = {xi[0], xi[1], xi[2]}, py[3] = {yi[0], yi[1], yi[2]};
        if (area2 < 0) {
            int32_t tx = px[1]; px[1] = px[2]; px[2] = tx;
            int32_t ty = py[1]; py[1] = py[2]; py[2] = ty;
        }
        for (int k = 0; k < 3; ++k) {
            int a = (k + 1) % 3, b = (k + 2) % 3;
            int64_t A = (int64_t)py[a] - py[b];
            int64_t Bc = (int64_t)px[b] - px[a];
            int64_t C = -(A * px[a] + Bc * py[a]);
            int tl = (A > 0) || (A == 0 && Bc > 0);
            int64_t Cpp = 128 * (A + Bc) + C - (tl ? 0 : 1);
            t->A[k] = (int32_t)A;
            t->B[k] = (int32_t)Bc;
            t->q[k] = Cpp >> 8; /* arithmetic shift = floor division */
        }
        int32_t xmin = px[0], xmax = px[0], ymin = py[0], ymax = py[0];
        for (int k = 1; k < 3; ++k) {
            if (px[k] < xmin) xmin = px[k];
            if (px[k] > xmax) xmax = px[k];
            if (py[k] < ymin) ymin = py[k];
            if (py[k] > ymax) ymax = py[k];
        }
        int cmin = (xmin + 127) >> 8, cmax = (xmax - 128) >> 8;
        int rmin = (ymin + 127) >> 8, rmax = (ymax - 128) >> 8;
        if (cmin < 0) cmin = 0;
        if (rmin < 0) rmin = 0;
        if (cmax > W - 1) cmax = W - 1;
        if (rmax > H - 1) rmax = H - 1;
        if (cmin > cmax || rmin > rmax) return;
        t->kind = 1;
        t->cmin = cmin; t->cmax = cmax; t->rmin = rmin; t->rmax = rmax;
        t->cref = cmin; t->rref = rmin;
    }
    t->zA = (float)gz[0]; t->zB = (float)gz[1]; t->zC = (float)gz[2];
    /* re-base q0,q1,S to (cref,rref):  C' = (A*cref + B*rref) + C  in double */
    {
        double cr = (double)t->cref, rr = (double)t->rref;
        t->q0[0] = (float)gq[0][0]; t->q0[1] = (float)gq[0][1];
        t->q0[2] = (float)((gq[0][0] * cr + gq[0][1] * rr) + gq[0][2]);
        t->q1[0] = (float)gq[1][0]; t->q1[1] = (float)gq[1][1];
        t->q1[2] = (float)((gq[1][0] * cr + gq[1][1] * rr) + gq[1][2]);
        t->s[0] = (float)gs[0]; t->s[1] = (float)gs[1];
        t->s[2] = (float)((gs[0] * cr + gs[1] * rr) + gs[2]);
    }
}

static inline int covers_normal(const Tri* t, int col, int row)
{
    for (int k = 0; k < 3; ++k) {
        int64_t n = (int64_t)t->A[k] * col + (int64_t)t->B[k] * row + t->q[k];
        if (n < 0) return 0;
    }
    return 1;
}

static inline int covers_hard(const Tri* t, int col, int row)
{
    double sum = 0.0;
    double qv[3];
    for (int k = 0; k < 3; ++k) {
        double tt = t->hq[k][1] * (double)row;
        tt = tt + t->hq[k][2];
        double u = t->hq[k][0] * (double)col;
        double v = u + tt;
        qv[k] = v;
        if (v > 0.0) continue;
        if (v == 0.0 && (t->hq[k][0] > 0.0 || (t->hq[k][0] == 0.0 && t->hq[k][1] > 0.0))) continue;
        return 0;
    }
    sum = (qv[0] + qv[1]) + qv[2];
    return sum > 0.0;
}

static inline uint32_t tri_depth_key(const Tri* t, int col, int row)
{
    float z;
    if (t->kind == 1) {
        z = fmaf(t->zA, (float)col, fmaf(t->zB, (float)row, t->zC));
    } else {
        double tt = t->hz[1] * (double)row;
        tt = tt + t->hz[2];
        double u = t->hz[0] * (double)col;
        z = (float)(u + tt);
    }
    return depth_key(z);
}

/* G: barycentrics and clip-w of face t at pixel (row,col), fp32 */
static inline void tri_gbuffer(const Tri* t, int col, int row, float out[4])
{
    float dc = (float)(col - t->cref), dr = (float)(row - t->rref);
    float S = fmaf(t->s[0], dc, fmaf(t->s[1], dr, t->s[2]));
    float cw = 1.0f / S;
    float q0 = fmaf(t->q0[0], dc, fmaf(t->q0[1], dr, t->q0[2]));
    float q1 = fmaf(t->q1[0], dc, fmaf(t->q1[1], dr, t->q1[2]));
    float b0 = q0 * cw, b1 = q1 * cw;
    out[0] = b0;
    out[1] = b1;
    out[2] = (1.0f - b0) - b1;
    out[3] = cw;
}

/* per-face setup of a whole batch, every (image, face) once, all threads: tris[B*F].  NULL if out of memory. */
static Tri* setup_batch(const float* vertices, const int32_t* faces, int B, int V, int F, int H, int W)
{
    Tri* tris = (Tri*)malloc(sizeof(Tri) * ((size_t)B * F > 0 ? (size_t)B * F : 1));
    if (!tris) return NULL;
    const long long total = (long long)B * F;
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < total; ++i) {
        const int b = (int)(i / F);
        setup_tri(vertices + (size_t)b * V * 4, faces + (size_t)i * 3, V, H, W, &tris[i]);
    }
    return tris;
}

/* visibility of rows [rb, re) of one image from its setup records tris[F]: face_ids / keys hold (re - rb) * W entries,
 * row rb first.  (Work is split over images and, when there are fewer images than threads, over bands of rows: a band
 * only needs the faces clipped to its rows, and the result per pixel does not depend on the split.) */
static void visibility_rows(int F, int W, const Tri* tris, int32_t* face_ids, uint32_t* keys, int rb, int re)
{
    for (int i = 0; i < (re - rb) * W; ++i) { face_ids[i] = -1; keys[i] = KEY_EMPTY; }
    for (int f = 0; f < F; ++f) {
        const Tri* t = &tris[f];
        if (t->kind == 0) continue;
        const int r0 = t->rmin > rb ? t->rmin : rb, r1 = t->rmax < re - 1 ? t->rmax : re - 1;
        for (int r = r0; r <= r1; ++r)
            for (int c = t->cmin; c <= t->cmax; ++c) {
                int in = (t->kind == 1) ? covers_normal(t, c, r) : covers_hard(t, c, r);
                if (!in) continue;
                uint32_t key = tri_depth_key(t, c, r);
                if (key < keys[(r - rb) * W + c]) { /* faces visited in ascending order: ties keep the earlier */
                    keys[(r - rb) * W + c] = key;
                    face_ids[(r - rb) * W + c] = f;
                }
            }
    }
}

/* how many bands of rows each image is cut into so that B * bands work items keep every thread busy */
static int bands_per_image(int B, int H)
{
    int threads = 1;
#ifdef _OPENMP
    threads = omp_get_max_threads();
#endif
    if (B <= 0 || B >= threads) return 1;
    int nb = (threads + B - 1) / B;
    if (nb > H) nb = H;
    return nb < 1 ? 1 : nb;
}

/* the reference's own greedy split of C (rasterise_ops.py:80-108) */
static int default_groups(int C, int* groups)
{
    int n = 0, begin = 0;
    if (C == 1 || C == 3) { groups[0] = C; return 1; }
    while (begin < C) {
        int wdt = (begin + 3 <= C) ? 3 : 1;
        groups[n++] = wdt;
        begin += wdt;
    }
    return n;
}

/* ------------------------------------------------------------------------------------- */
/* exported API (mirrors include/dirt_b200.h, host pointers)                              */
/* ------------------------------------------------------------------------------------- */

int dirt_oracle_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

void dirt_oracle_set_threads(int n)
{
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

/* face_ids [B,H,W] and gbuffer [B,H,W,4] (either may be NULL) */
int dirt_oracle_visibility(const float* vertices, const int32_t* faces, int32_t* face_ids, float* gbuffer,
                           int B, int H, int W, int V, int F)
{
    if (B < 0 || H <= 0 || W <= 0 || V < 0 || F < 0) return -1;
    int fail = 0;
    const int NB = bands_per_image(B, H);
    Tri* all_tris = setup_batch(vertices, faces, B, V, F, H, W);
    if (!all_tris) return -2;
#pragma omp parallel for schedule(dynamic, 1)
    for (int item = 0; item < B * NB; ++item) {
        const int b = item / NB, band = item % NB;
        const int rb = (int)((long long)H * band / NB), re = (int)((long long)H * (band + 1) / NB);
        const Tri* tris = all_tris + (size_t)b * F;
        int32_t* ids = (int32_t*)malloc(sizeof(int32_t) * (size_t)(re - rb) * W);
        uint32_t* keys = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(re - rb) * W);
        if (!ids || !keys) { fail = 1; free(ids); free(keys); continue; }
        visibility_rows(F, W, tris, ids, keys, rb, re);
        if (face_ids) memcpy(face_ids + ((size_t)b * H + rb) * W, ids, sizeof(int32_t) * (size_t)(re - rb) * W);
        if (gbuffer)
            for (int r = rb; r < re; ++r)
                for (int c = 0; c < W; ++c) {
                    float* g = gbuffer + (((size_t)b * H + r) * W + c) * 4;
                    int f = ids[(r - rb) * W + c];
                    if (f < 0) { g[0] = g[1] = g[2] = -1.0f; g[3] = INFINITY; }
                    else tri_gbuffer(&tris[f], c, r, g);
                }
        free(ids); free(keys);
    }
    free(all_tris);
    return fail ? -2 : 0;
}

int dirt_oracle_forward(const float* background, const float* vertices, const float* vertex_colors,
                        const int32_t* faces, float* pixels, int32_t* face_ids_out,
                        int B, int H, int W, int C, int V, int F)
{
    if (B < 0 || H <= 0 || W <= 0 || C <= 0 || V < 0 || F < 0) return -1;
    int fail = 0;
    const int NB = bands_per_image(B, H);
    Tri* all_tris = setup_batch(vertices, faces, B, V, F, H, W);
    if (!all_tris) return -2;
#pragma omp parallel for schedule(dynamic, 1)
    for (int item = 0; item < B * NB; ++item) {
        const int b = item / NB, band = item % NB;
        const int rb = (int)((long long)H * band / NB), re = (int)((long long)H * (band + 1) / NB);
        const Tri* tris = all_tris + (size_t)b * F;
        int32_t* ids = (int32_t*)malloc(sizeof(int32_t) * (size_t)(re - rb) * W);
        uint32_t* keys = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(re - rb) * W);
        if (!ids || !keys) { fail = 1; free(ids); free(keys); continue; }
        visibility_rows(F, W, tris, ids, keys, rb, re);
        const float* cols = vertex_colors + (size_t)b * V * C;
        for (int r = rb; r < re; ++r)
            for (int c = 0; c < W; ++c) {
                size_t pix = ((size_t)b * H + r) * W + c;
                int f = ids[(r - rb) * W + c];
                if (f < 0) {
                    for (int ch = 0; ch < C; ++ch) pixels[pix * C + ch] = background[pix * C + ch];
                } else {
                    float g[4];
                    tri_gbuffer(&tris[f], c, r, g);
                    const Tri* t = &tris[f];
                    for (int ch = 0; ch < C; ++ch) {
                        /* c2 + b0*(c0-c2) + b1*(c1-c2): exact when the three vertex colours are equal, as
                         * tests/square_test.py requires of the hardware interpolator */
                        double c0 = cols[(size_t)t->v[0] * C + ch], c1 = cols[(size_t)t->v[1] * C + ch];
                        double c2 = cols[(size_t)t->v[2] * C + ch];
                        double acc = c2 + ((double)g[0] * (c0 - c2) + (double)g[1] * (c1 - c2));
                        pixels[pix * C + ch] = (float)acc;
                    }
                }
            }
        if (face_ids_out) memcpy(face_ids_out + ((size_t)b * H + rb) * W, ids, sizeof(int32_t) * (size_t)(re - rb) * W);
        free(ids); free(keys);
    }
    free(all_tris);
    return fail ? -2 : 0;
}

/* assemble_grads (csrc/rasterise_grad_egl.cu:93-236) for one channel group of one image.
 * pixels/grad_pixels/grad_background are the fused [B,H,W,C] tensors, the group is
 * channels [c0, c0+n).  Decision quantities (Scharr sums, L1, clip_w) are fp32 in the
 * order the reference writes them; accumulations are double. */
typedef struct { float x, y, z; } V3;

static inline V3 group_at(const float* pixels, int b, int r, int c, int B, int H, int W, int C, int c0, int n)
{
    /* at(): nearest edge pixel for out-of-bounds (csrc/rasterise_grad_egl.cu:113-124);
     * always three components.  For a 1-channel group the reference indexes a contiguous
     * [B,H,W,1] tensor with channel 1 and 2, i.e. the next two pixels in flat order
     * (SURVEY Appendix A.4.1); reads past the end of the tensor are defined as 0 here. */
    if (r < 0) r = 0; if (r > H - 1) r = H - 1;
    if (c < 0) c = 0; if (c > W - 1) c = W - 1;
    size_t lin = ((size_t)b * H + r) * W + c;
    V3 v;
    if (n == 3) {
        v.x = pixels[lin * C + c0];
        v.y = pixels[lin * C + c0 + 1];
        v.z = pixels[lin * C + c0 + 2];
    } else {
        size_t total = (size_t)B * H * W;
        v.x = pixels[lin * C + c0];
        v.y = (lin + 1 < total) ? pixels[(lin + 1) * C + c0] : 0.0f;
        v.z = (lin + 2 < total) ? pixels[(lin + 2) * C + c0] : 0.0f;
    }
    return v;
}

static inline float scharr_comp(float nn, float np, float pn, float pp, float mn, float mp)
{
    /* (a + b - c - d) * (3/32) + (e - f) * (10/32) (csrc/rasterise_grad_egl.cu:126-127), the sum of products
     * contracted the way nvcc contracts it when it compiles the reference file itself:
     *     FMUL t, (e - f), 0.3125 ;  FFMA r, (a + b - c - d), 0.09375, t
     * (oracle/_ref, SASS: make -C oracle ref-sass) */
    float X = ((nn + np) - pn) - pp;
    float Y = mn - mp;
    return fmaf(X, 0.09375f, Y * 0.3125f);
}

static void backward_image_group(const float* verts, const Tri* tris, const int32_t* ids_rows, int rb,
                                 const float* pixels, const float* grad_pixels,
                                 double* gverts /*[V,4]*/, int b, int B, int H, int W, int C, int c0, int n, int r0, int r1,
                                 uint8_t* codes /*[B,H,W] of this group, or NULL*/)
{
    /* rows [r0, r1) of the image; ids_rows holds the visibility buffer from row rb on (rb <= r0 - 1 unless r0 == 0).
     * `codes` receives the dilation code of every pixel (include/dirt_b200.h, dirt_rasterise_backward_deterministic):
     * bits 0-1  0: no position term, 1: the own face takes it, 2 / 3: the neighbour of the first / second attempt does
     * (the reference's debug_thingy[..., 0] = 1e-2, :172); bit 2: the preferred step runs along the row (interior pixels) */
#define IDS(r_, c_) ids_rows[((r_) - rb) * W + (c_)]
    for (int r = r0; r < r1; ++r)
        for (int c = 0; c < W; ++c) {
            /* at(ox,oy) is image (row r - oy, col c + ox) */
#define AT(ox, oy) group_at(pixels, b, r - (oy), c + (ox), B, H, W, C, c0, n)
            V3 a_mm = AT(-1, -1), a_mp = AT(-1, +1), a_pm = AT(+1, -1), a_pp = AT(+1, +1);
            V3 a_m0 = AT(-1, 0), a_p0 = AT(+1, 0), a_0m = AT(0, -1), a_0p = AT(0, +1);
#undef AT
            float sx[3], sy[3];
            /* scharr_x = (at(-1,-1) + at(-1,+1) - at(+1,-1) - at(+1,+1))*3/32 + (at(-1,0) - at(+1,0))*10/32 */
            sx[0] = scharr_comp(a_mm.x, a_mp.x, a_pm.x, a_pp.x, a_m0.x, a_p0.x);
            sx[1] = scharr_comp(a_mm.y, a_mp.y, a_pm.y, a_pp.y, a_m0.y, a_p0.y);
            sx[2] = scharr_comp(a_mm.z, a_mp.z, a_pm.z, a_pp.z, a_m0.z, a_p0.z);
            /* scharr_y = (at(-1,-1) + at(+1,-1) - at(-1,+1) - at(+1,+1))*3/32 + (at(0,-1) - at(0,+1))*10/32 */
            sy[0] = scharr_comp(a_mm.x, a_pm.x, a_mp.x, a_pp.x, a_0m.x, a_0p.x);
            sy[1] = scharr_comp(a_mm.y, a_pm.y, a_mp.y, a_pp.y, a_0m.y, a_0p.y);
            sy[2] = scharr_comp(a_mm.z, a_pm.z, a_mp.z, a_pp.z, a_0m.z, a_0p.z);

            int f = IDS(r, c);
            float g[4] = {-1.0f, -1.0f, -1.0f, INFINITY};
            if (f >= 0) tri_gbuffer(&tris[f], c, r, g);

            /* dilation (:155-194), interior pixels only */
            int code = 1;
            if (c > 0 && r > 0 && c < W - 1 && r < H - 1) {
                float l1x = (fabsf(sx[0]) + fabsf(sx[1])) + fabsf(sx[2]);
                float l1y = (fabsf(sy[0]) + fabsf(sy[1])) + fabsf(sy[2]);
                int dx = (l1x > l1y) ? 1 : 0, dy = (l1x > l1y) ? 0 : 1; /* buffer (GL, y-up) orientation */
                if (dx) code |= 4;
                if ((c + r) % 2 == 1) { dx = -dx; dy = -dy; }
                for (int attempt = 0; attempt < 2; ++attempt) {
                    int nc = c + dx, nr = r - dy; /* buffer_y + dy is image row r - dy */
                    int fn = IDS(nr, nc);
                    if (fn >= 0) {
                        const Tri* tn = &tris[fn];
                        int differs = (f < 0) || tn->v[0] != tris[f].v[0] || tn->v[1] != tris[f].v[1] ||
                                      tn->v[2] != tris[f].v[2];
                        float gn[4];
                        tri_gbuffer(tn, nc, nr, gn);
                        if (differs && g[3] > gn[3]) {
                            g[0] = gn[0]; g[1] = gn[1]; g[2] = gn[2]; g[3] = gn[3];
                            f = fn;
                            code += 1 + attempt;
                            break;
                        }
                    }
                    dx = -dx; dy = -dy;
                }
            }

            if (codes) codes[((size_t)b * H + r) * W + c] = (uint8_t)(f >= 0 ? code : 0);
            if (f >= 0) { /* position gradients (:196-232) */
                const Tri* t = &tris[f];
                size_t pix = ((size_t)b * H + r) * W + c;
                double dLdx = 0.0, dLdy = 0.0;
                for (int ch = 0; ch < n; ++ch) {
                    double gp = grad_pixels[pix * C + c0 + ch];
                    dLdx += gp * sx[ch];
                    dLdy += gp * sy[ch];
                }
                double clip_x = 0.0, clip_y = 0.0;
                for (int k = 0; k < 3; ++k) {
                    clip_x += (double)g[k] * verts[(size_t)t->v[k] * 4 + 0];
                    clip_y += (double)g[k] * verts[(size_t)t->v[k] * 4 + 1];
                }
                double cw = g[3];
                double dxv_dxc = 0.5 * W / cw, dyv_dyc = 0.5 * H / cw;
                double dxv_dwc = -0.5 * W * clip_x / (cw * cw), dyv_dwc = -0.5 * H * clip_y / (cw * cw);
                for (int k = 0; k < 3; ++k) {
                    double ax = dLdx * g[k], ay = dLdy * g[k];
                    gverts[(size_t)t->v[k] * 4 + 0] += ax * dxv_dxc;
                    gverts[(size_t)t->v[k] * 4 + 1] += ay * dyv_dyc;
                    gverts[(size_t)t->v[k] * 4 + 3] += ax * dxv_dwc + ay * dyv_dwc;
                }
            }
        }
#undef IDS
}

/* dirt_oracle_backward with the dilation decisions: `codes` (NULL, or uint8 [n_groups, B, H, W] with one plane per
 * channel group in call order) gets every pixel's dilation code (backward_image_group) */
int dirt_oracle_backward_ex(const float* vertices, const int32_t* faces, const float* pixels,
                            const float* grad_pixels, float* grad_background, float* grad_vertices,
                            float* grad_vertex_colors, int B, int H, int W, int C, int V, int F,
                            const int* channel_groups, int n_groups, uint8_t* codes)
{
    if (B < 0 || H <= 0 || W <= 0 || C <= 0 || V < 0 || F < 0) return -1;
    int* groups = (int*)malloc(sizeof(int) * (size_t)(C + 1));
    if (!groups) return -2;
    int ng;
    if (channel_groups && n_groups > 0) {
        int sum = 0;
        for (int i = 0; i < n_groups; ++i) {
            if (channel_groups[i] != 1 && channel_groups[i] != 3) { free(groups); return -4; }
            groups[i] = channel_groups[i];
            sum += channel_groups[i];
        }
        if (sum != C) { free(groups); return -4; }
        ng = n_groups;
    } else {
        ng = default_groups(C, groups);
    }
    int fail = 0;
    /* work items: (image, band of rows); every item sums into its own double accumulators, which are added up per image
     * in band order afterwards (deterministic for a given thread count) */
    const int NB = bands_per_image(B, H);
    const size_t nv = (size_t)(V > 0 ? V : 1);
    double* gv_all = (double*)calloc((size_t)(B > 0 ? B : 1) * NB * nv * 4, sizeof(double));
    double* gc_all = (double*)calloc((size_t)(B > 0 ? B : 1) * NB * nv * C, sizeof(double));
    Tri* all_tris = setup_batch(vertices, faces, B, V, F, H, W);
    if (!gv_all || !gc_all || !all_tris) { free(gv_all); free(gc_all); free(all_tris); free(groups); return -2; }
#pragma omp parallel for schedule(dynamic, 1)
    for (int item = 0; item < B * NB; ++item) {
        const int b = item / NB, band = item % NB;
        const int r0 = (int)((long long)H * band / NB), r1 = (int)((long long)H * (band + 1) / NB);
        const int rb = r0 > 0 ? r0 - 1 : 0, re = r1 < H ? r1 + 1 : H;   /* the dilation looks one row up and down */
        const Tri* tris = all_tris + (size_t)b * F;
        int32_t* ids = (int32_t*)malloc(sizeof(int32_t) * (size_t)(re - rb) * W);
        uint32_t* keys = (uint32_t*)malloc(sizeof(uint32_t) * (size_t)(re - rb) * W);
        if (!ids || !keys) {
            fail = 1; free(ids); free(keys);
            continue;
        }
        double* gv = gv_all + (size_t)item * nv * 4;
        double* gc = gc_all + (size_t)item * nv * C;
        const float* verts = vertices + (size_t)b * V * 4;
        visibility_rows(F, W, tris, ids, keys, rb, re);
        /* colour gradients and background gradient (:135-148): undilated barycentrics, all channels */
        for (int r = r0; r < r1; ++r)
            for (int c = 0; c < W; ++c) {
                size_t pix = ((size_t)b * H + r) * W + c;
                int f = ids[(r - rb) * W + c];
                if (f >= 0) {
                    float g[4];
                    tri_gbuffer(&tris[f], c, r, g);
                    for (int k = 0; k < 3; ++k)
                        for (int ch = 0; ch < C; ++ch)
                            gc[(size_t)tris[f].v[k] * C + ch] += (double)grad_pixels[pix * C + ch] * g[k];
                    for (int ch = 0; ch < C; ++ch) grad_background[pix * C + ch] = 0.0f;
                } else {
                    for (int ch = 0; ch < C; ++ch) grad_background[pix * C + ch] = grad_pixels[pix * C + ch];
                }
            }
        int c0 = 0;
        for (int gi = 0; gi < ng; ++gi) {
            backward_image_group(verts, tris, ids, rb, pixels, grad_pixels, gv, b, B, H, W, C, c0, groups[gi], r0, r1,
                                 codes ? codes + (size_t)gi * B * H * W : NULL);
            c0 += groups[gi];
        }
        free(ids); free(keys);
    }
    free(all_tris);
#pragma omp parallel for schedule(static)
    for (int b = 0; b < B; ++b) {
        for (size_t i = 0; i < (size_t)V * 4; ++i) {
            double acc = 0.0;
            for (int band = 0; band < NB; ++band) acc += gv_all[((size_t)b * NB + band) * nv * 4 + i];
            grad_vertices[(size_t)b * V * 4 + i] = (float)acc;
        }
        for (size_t i = 0; i < (size_t)V * C; ++i) {
            double acc = 0.0;
            for (int band = 0; band < NB; ++band) acc += gc_all[((size_t)b * NB + band) * nv * C + i];
            grad_vertex_colors[(size_t)b * V * C + i] = (float)acc;
        }
    }
    free(gv_all); free(gc_all);
    free(groups);
    return fail ? -2 : 0;
}

int dirt_oracle_backward(const float* vertices, const int32_t* faces, const float* pixels,
                         const float* grad_pixels, float* grad_background, float* grad_vertices,
                         float* grad_vertex_colors, int B, int H, int W, int C, int V, int F,
                         const int* channel_groups, int n_groups)
{
    return dirt_oracle_backward_ex(vertices, faces, pixels, grad_pixels, grad_background, grad_vertices,
                                   grad_vertex_colors, B, H, W, C, V, F, channel_groups, n_groups, NULL);
}

/* debug: per-face setup records of one image, for comparing the CUDA setup kernel bit for bit */
int dirt_oracle_setup(const float* vertices /*[V,4]*/, const int32_t* faces /*[F,3]*/, TriExport* out,
                      int H, int W, int V, int F)
{
    for (int f = 0; f < F; ++f) {
        Tri t;
        setup_tri(vertices, faces + (size_t)f * 3, V, H, W, &t);
        TriExport* e = &out[f];
        memset(e, 0, sizeof(*e));
        e->kind = t.kind;
        for (int k = 0; k < 3; ++k) { e->A[k] = t.A[k]; e->B[k] = t.B[k]; e->q[k] = t.q[k]; }
        e->z[0] = t.zA; e->z[1] = t.zB; e->z[2] = t.zC;
        for (int k = 0; k < 3; ++k) { e->q0[k] = t.q0[k]; e->q1[k] = t.q1[k]; e->s[k] = t.s[k]; }
        e->cref = t.cref; e->rref = t.rref;
        e->bbox[0] = t.cmin; e->bbox[1] = t.rmin; e->bbox[2] = t.cmax; e->bbox[3] = t.rmax;
    }
    return 0;
}
