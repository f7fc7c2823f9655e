/*
 * oracle.c -- CPU restatement of the reference rasterizer's hot path, in plain C.
 *
 * TEST INFRASTRUCTURE ONLY.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load
 * this; the product (rade-gs_b200/) never does and has no CPU path.
 *
 * It restates, serially and without atomics, what the reference computes (paths relative to
 * submodules/diff-gaussian-rasterization/cuda_rasterizer/ of the reference):
 *   orc_preprocess           forward.cu:270-304 (cov3D), :77-264 (cov2D, planes, normal), :23-74 (SH), :307-423
 *   orc_eig_sym3             auxiliary.h:182-401 (Householder + QL with absolute 1e-7 tests)
 *   orc_binning              rasterizer_impl.cu:70-111 (keys), :373-381 (stable sort), :151-173 (ranges)
 *   orc_render_forward       forward.cu:428-693
 *   orc_render_backward      backward.cu:631-1016  (scatter sums in double, one thread, deterministic)
 *   orc_preprocess_backward  backward.cu:145-488, :560-628, :21-140, :492-555
 *                            including the dL_dconic-for-conic_opacity aliasing (rasterizer_impl.cu:569)
 *   orc_inte_geometry        forward.cu:187-235 (computeCov2D<INTE>: inverse ray-space covariance, well-conditioned flag)
 *   orc_integrate            forward.cu:857-900 (points), rasterizer_impl.cu:114-145 (point -> tile), forward.cu:938-1372
 *
 * Parity pin: tests/test_oracle_golden.py checks every function against tests/golden/<case>.npz, which were
 * produced by the unmodified reference CUDA build (tools/gen_golden.py).
 *
 * Arithmetic is float with the same double-promoted sub-expressions as the reference; gcc is run with
 * -ffp-contract=off, so results differ from the CUDA builds (which contract to FMA) in the last bits only.
 * Matrices are column-major 3x3 like glm: m.c[col][row].
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define TILE 16

typedef struct { float c[3][3]; } m3;   /* c[col][row] */
typedef struct { float v[3]; } v3;

static m3 m3_make(float a0, float a1, float a2, float b0, float b1, float b2, float c0, float c1, float c2) {
	m3 m = {{{a0, a1, a2}, {b0, b1, b2}, {c0, c1, c2}}};
	return m;
}
static m3 m3_t(m3 a) {
	m3 r;
	for (int c = 0; c < 3; c++) for (int k = 0; k < 3; k++) r.c[c][k] = a.c[k][c];
	return r;
}
static m3 m3_mul(m3 a, m3 b) {
	m3 r;
	for (int c = 0; c < 3; c++)
		for (int k = 0; k < 3; k++) r.c[c][k] = a.c[0][k] * b.c[c][0] + a.c[1][k] * b.c[c][1] + a.c[2][k] * b.c[c][2];
	return r;
}
static v3 m3_mulv(m3 a, v3 x) {
	v3 r;
	for (int k = 0; k < 3; k++) r.v[k] = a.c[0][k] * x.v[0] + a.c[1][k] * x.v[1] + a.c[2][k] * x.v[2];
	return r;
}
static m3 m3_scale(m3 a, float s) { m3 r; for (int c = 0; c < 3; c++) for (int k = 0; k < 3; k++) r.c[c][k] = a.c[c][k] * s; return r; }
static m3 m3_div(m3 a, float s) { m3 r; for (int c = 0; c < 3; c++) for (int k = 0; k < 3; k++) r.c[c][k] = a.c[c][k] / s; return r; }
static m3 m3_add(m3 a, m3 b) { m3 r; for (int c = 0; c < 3; c++) for (int k = 0; k < 3; k++) r.c[c][k] = a.c[c][k] + b.c[c][k]; return r; }
static m3 m3_outer(v3 col, v3 row) { m3 r; for (int c = 0; c < 3; c++) for (int k = 0; k < 3; k++) r.c[c][k] = col.v[k] * row.v[c]; return r; }
static m3 m3_zero(void) { m3 r; memset(&r, 0, sizeof r); return r; }
static v3 v3_make(float x, float y, float z) { v3 r = {{x, y, z}}; return r; }
static v3 v3_add(v3 a, v3 b) { return v3_make(a.v[0] + b.v[0], a.v[1] + b.v[1], a.v[2] + b.v[2]); }
static v3 v3_sub(v3 a, v3 b) { return v3_make(a.v[0] - b.v[0], a.v[1] - b.v[1], a.v[2] - b.v[2]); }
static v3 v3_scale(v3 a, float s) { return v3_make(a.v[0] * s, a.v[1] * s, a.v[2] * s); }
static v3 v3_div(v3 a, float s) { return v3_make(a.v[0] / s, a.v[1] / s, a.v[2] / s); }
static float v3_dot(v3 a, v3 b) { float t0 = a.v[0] * b.v[0], t1 = a.v[1] * b.v[1], t2 = a.v[2] * b.v[2]; return t0 + t1 + t2; }
static v3 v3_normalize(v3 a) { return v3_scale(a, 1.0f / sqrtf(v3_dot(a, a))); }
static float fminf2(float a, float b) { return a < b ? a : b; }
static float fmaxf2(float a, float b) { return a > b ? a : b; }

/* auxiliary.h:74-113.  nvcc contracts a*b + c*d + e*f + g into mul, fma, fma, add (default -fmad=true); the
 * result decides the depth bits of the sort keys and the pixel position, so the same contraction (SASS: FMUL b*y; FFMA a*x+.; FFMA c*z+.; FADD +d) is spelled
 * out here with fmaf() -- verified bit-exact against the golden fixtures (tests/test_oracle_golden.py). */
static float dot3_fma(float a, float x, float b, float y, float c, float z, float d) { return fmaf(c, z, fmaf(a, x, b * y)) + d; }
static void xf4x3(const float* p, const float* m, float* o) {
	o[0] = dot3_fma(m[0], p[0], m[4], p[1], m[8], p[2], m[12]);
	o[1] = dot3_fma(m[1], p[0], m[5], p[1], m[9], p[2], m[13]);
	o[2] = dot3_fma(m[2], p[0], m[6], p[1], m[10], p[2], m[14]);
}
static void xf4x4(const float* p, const float* m, float* o) {
	xf4x3(p, m, o);
	o[3] = dot3_fma(m[3], p[0], m[7], p[1], m[11], p[2], m[15]);
}
static void xfvec4x3T(const float* p, const float* m, float* o) {
	o[0] = m[0] * p[0] + m[1] * p[1] + m[2] * p[2];
	o[1] = m[4] * p[0] + m[5] * p[1] + m[6] * p[2];
	o[2] = m[8] * p[0] + m[9] * p[1] + m[10] * p[2];
}
/* auxiliary.h:57-60: unsuffixed literals -> double */
static float ndc2pix(float v, int S) { return (float)(((v + 1.0) * S - 1.0) * 0.5); }
/* auxiliary.h:62-72 */
static void get_rect(float px, float py, int r, int gx, int gy, int* x0, int* y0, int* x1, int* y1) {
	int a;
	a = (int)((px - r) / TILE); *x0 = a < 0 ? 0 : (a > gx ? gx : a);
	a = (int)((py - r) / TILE); *y0 = a < 0 ? 0 : (a > gy ? gy : a);
	a = (int)((px + r + TILE - 1) / TILE); *x1 = a < 0 ? 0 : (a > gx ? gx : a);
	a = (int)((py + r + TILE - 1) / TILE); *y1 = a < 0 ? 0 : (a > gy ? gy : a);
}

/* ---- symmetric 3x3 eigen-solver, auxiliary.h:182-401 ------------------------------------------------------ */
static const float EPS7 = 0.0000001f;
static int near0(float x) { return fabsf(x) <= EPS7; }
static float pyth(float a, float b) {
	float aa = fabsf(a), ab = fabsf(b);
	if (aa > ab) { ab /= aa; ab *= ab; return aa * sqrtf(1.0f + ab); }
	if (near0(ab)) return 0.0f;
	aa /= ab; aa *= aa; return ab * sqrtf(1.0f + aa);
}
/* returns 3 on success, 0 when a QL sweep exceeds 30 iterations; vec columns are eigenvectors */
int orc_eig_sym3(const float* cov6, float* lam, float* vec_colmajor) {
	enum { D = 3 };
	float a[D * D], d[D], e[D];
	const float full[9] = {cov6[0], cov6[1], cov6[2], cov6[1], cov6[3], cov6[4], cov6[2], cov6[4], cov6[5]};
	memcpy(a, full, sizeof a);
	int l, k, j, i;
	float scale, hh, h, g, f;
	for (i = D; i >= 2; i--) {
		l = i - 1; h = scale = 0;
		if (l > 1) {
			for (k = 1; k <= l; k++) scale += fabsf(a[(i - 1) * D + (k - 1)]);
			if (near0(scale)) e[i - 1] = a[(i - 1) * D + (l - 1)];
			else {
				for (k = 1; k <= l; k++) { a[(i - 1) * D + (k - 1)] /= scale; h += a[(i - 1) * D + (k - 1)] * a[(i - 1) * D + (k - 1)]; }
				f = a[(i - 1) * D + (l - 1)];
				g = (f >= 0) ? -sqrtf(h) : sqrtf(h);
				e[i - 1] = scale * g; h -= f * g; a[(i - 1) * D + (l - 1)] = f - g; f = 0;
				for (j = 1; j <= l; j++) {
					a[(j - 1) * D + (i - 1)] = a[(i - 1) * D + (j - 1)] / h; g = 0;
					for (k = 1; k <= j; k++) g += a[(j - 1) * D + (k - 1)] * a[(i - 1) * D + (k - 1)];
					for (k = j + 1; k <= l; k++) g += a[(k - 1) * D + (j - 1)] * a[(i - 1) * D + (k - 1)];
					e[j - 1] = g / h; f += e[j - 1] * a[(i - 1) * D + (j - 1)];
				}
				hh = f / (h + h);
				for (j = 1; j <= l; j++) {
					f = a[(i - 1) * D + (j - 1)]; e[j - 1] = g = e[j - 1] - hh * f;
					for (k = 1; k <= j; k++) a[(j - 1) * D + (k - 1)] -= (f * e[k - 1] + g * a[(i - 1) * D + (k - 1)]);
				}
			}
		} else e[i - 1] = a[(i - 1) * D + (l - 1)];
		d[i - 1] = h;
	}
	d[0] = 0; e[0] = 0;
	for (i = 1; i <= D; i++) {
		l = i - 1;
		if (!near0(d[i - 1])) {
			for (j = 1; j <= l; j++) {
				g = 0;
				for (k = 1; k <= l; k++) g += a[(i - 1) * D + (k - 1)] * a[(k - 1) * D + (j - 1)];
				for (k = 1; k <= l; k++) a[(k - 1) * D + (j - 1)] -= g * a[(k - 1) * D + (i - 1)];
			}
		}
		d[i - 1] = a[(i - 1) * D + (i - 1)]; a[(i - 1) * D + (i - 1)] = 1;
		for (j = 1; j <= l; j++) a[(j - 1) * D + (i - 1)] = a[(i - 1) * D + (j - 1)] = 0;
	}
	int m, iter;
	float s, r, p, c, b;
	for (i = 2; i <= D; i++) e[i - 2] = e[i - 1];
	e[D - 1] = 0;
	for (l = 1; l <= D; l++) {
		iter = 0;
		do {
			for (m = l; m <= D - 1; m++) if (near0(fabsf(e[m - 1]))) break;
			if (m != l) {
				if (iter++ == 30) return 0;
				g = (d[l] - d[l - 1]) / (2 * e[l - 1]);
				r = pyth(g, 1);
				g = d[m - 1] - d[l - 1] + e[l - 1] / (g + (g >= 0 ? fabsf(r) : -fabsf(r)));
				s = c = 1; p = 0;
				for (i = m - 1; i >= l; i--) {
					f = s * e[i - 1]; b = c * e[i - 1];
					e[i] = r = pyth(f, g);
					if (near0(r)) { d[i] -= p; e[m - 1] = 0; break; }
					s = f / r; c = g / r; g = d[i] - p;
					r = (d[i - 1] - g) * s + 2 * c * b;
					d[i] = g + (p = s * r); g = c * r - b;
					for (k = 1; k <= D; k++) {
						f = a[(k - 1) * D + i];
						a[(k - 1) * D + i] = s * a[(k - 1) * D + (i - 1)] + c * f;
						a[(k - 1) * D + (i - 1)] = c * a[(k - 1) * D + (i - 1)] - s * f;
					}
				}
				if (near0(r) && i >= l) continue;
				d[l - 1] -= p; e[l - 1] = g; e[m - 1] = 0;
			}
		} while (m != l);
	}
	for (i = 0; i < D; i++) lam[i] = d[i];
	for (i = 0; i < D; i++) for (j = 0; j < D; j++) vec_colmajor[i * 3 + j] = a[j * D + i];
	return D;
}

typedef struct {
	m3 inv, E; float lam[3]; int min_id, well, solved;
} sig_inv;
static sig_inv sigma_inverse(const float* cov6) {
	sig_inv s; float vec[9];
	s.solved = orc_eig_sym3(cov6, s.lam, vec) != 0;
	for (int c = 0; c < 3; c++) for (int k = 0; k < 3; k++) s.E.c[c][k] = vec[c * 3 + k];
	const float* l = s.lam;
	s.min_id = l[0] > l[1] ? (l[1] > l[2] ? 2 : 1) : (l[0] > l[2] ? 2 : 0);
	s.well = l[s.min_id] > 0.00000001f;
	if (s.well) {
		m3 dg = m3_make(1 / l[0], 0, 0, 0, 1 / l[1], 0, 0, 0, 1 / l[2]);
		s.inv = m3_mul(m3_mul(s.E, dg), m3_t(s.E));
	} else {
		v3 em = v3_make(s.E.c[s.min_id][0], s.E.c[s.min_id][1], s.E.c[s.min_id][2]);
		s.inv = m3_outer(em, em);
	}
	return s;
}

/* forward.cu:270-304 */
static void cov3d_from_scale_rot(const float* sc, float mod, const float* q, float* cov6) {
	m3 S = m3_make(mod * sc[0], 0, 0, 0, mod * sc[1], 0, 0, 0, mod * sc[2]);
	float r = q[0], x = q[1], y = q[2], z = q[3];
	m3 R = m3_make(1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y),
	               2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x),
	               2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y));
	m3 M = m3_mul(S, R);
	m3 Sg = m3_mul(m3_t(M), M);
	cov6[0] = Sg.c[0][0]; cov6[1] = Sg.c[0][1]; cov6[2] = Sg.c[0][2]; cov6[3] = Sg.c[1][1]; cov6[4] = Sg.c[1][2]; cov6[5] = Sg.c[2][2];
}

static const float SH_C0 = 0.28209479177387814f, SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                               -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};

typedef struct {
	int P, D, M, W, H;
	float tan_fovx, tan_fovy, kernel_size, scale_modifier;
	const float *means3D, *opacities, *shs, *colors_precomp, *scales, *rotations, *cov3D_precomp;
	const float *viewmatrix, *projmatrix, *cam_pos;
} orc_scene;

/* per-Gaussian state, SoA like the reference's GeometryState (rasterizer_impl.cu:190-210) */
typedef struct {
	int* radii; float* means2D; float* depths; float* conic_opacity; float* rgb; uint8_t* clamped; float* cov3D;
	float* ts; float* ray_planes; float* camera_planes; float* normals; float* view_points; uint32_t* tiles_touched;
} orc_geom;

/* forward.cu:307-423 (+ helpers) */
void orc_preprocess(const orc_scene* s, orc_geom* g) {
	const int gx = (s->W + TILE - 1) / TILE, gy = (s->H + TILE - 1) / TILE;
	const float focal_y = s->H / (2.0f * s->tan_fovy), focal_x = s->W / (2.0f * s->tan_fovx);
	const float* V = s->viewmatrix;
	for (int idx = 0; idx < s->P; idx++) {
		g->radii[idx] = 0; g->tiles_touched[idx] = 0;
		const float* po = s->means3D + 3 * idx;
		float pv[3]; xf4x3(po, V, pv);
		if (pv[2] <= 0.2f) continue;
		float ph[4]; xf4x4(po, s->projmatrix, ph);
		float pw = 1.0f / (ph[3] + 0.0000001f);
		float pp[3] = {ph[0] * pw, ph[1] * pw, ph[2] * pw};
		float* cov6 = g->cov3D + 6 * idx;
		if (s->cov3D_precomp) memcpy(cov6, s->cov3D_precomp + 6 * idx, 6 * sizeof(float));
		else cov3d_from_scale_rot(s->scales + 3 * idx, s->scale_modifier, s->rotations + 4 * idx, cov6);

		/* computeCov2D, forward.cu:85-124 */
		float t[3] = {pv[0], pv[1], pv[2]};
		const float limx = 1.3f * s->tan_fovx, limy = 1.3f * s->tan_fovy;
		float txtz = t[0] / t[2], tytz = t[1] / t[2];
		t[0] = fminf2(limx, fmaxf2(-limx, txtz)) * t[2];
		t[1] = fminf2(limy, fmaxf2(-limy, tytz)) * t[2];
		txtz = t[0] / t[2]; tytz = t[1] / t[2];
		m3 J = m3_make(focal_x / t[2], 0.0f, -(focal_x * t[0]) / (t[2] * t[2]), 0.0f, focal_y / t[2], -(focal_y * t[1]) / (t[2] * t[2]), 0, 0, 0);
		m3 Wm = m3_make(V[0], V[4], V[8], V[1], V[5], V[9], V[2], V[6], V[10]);
		m3 T = m3_mul(Wm, J);
		m3 Vrk = m3_make(cov6[0], cov6[1], cov6[2], cov6[1], cov6[3], cov6[4], cov6[2], cov6[4], cov6[5]);
		m3 cov = m3_mul(m3_mul(m3_t(T), m3_t(Vrk)), T);
		const float ks = s->kernel_size;
		float cov2[3] = {cov.c[0][0] + ks, cov.c[0][1], cov.c[1][1] + ks};
		const float det_0 = (float)fmax(1e-6, (double)(cov.c[0][0] * cov.c[1][1] - cov.c[0][1] * cov.c[0][1]));
		const float det_1 = (float)fmax(1e-6, (double)((cov.c[0][0] + ks) * (cov.c[1][1] + ks) - cov.c[0][1] * cov.c[0][1]));
		float coef = (float)sqrt(det_0 / (det_1 + 1e-6) + 1e-6);
		if (det_0 <= 1e-6 || det_1 <= 1e-6) coef = 0.0f;

		/* planes / normal, forward.cu:135-262; written before the early-outs below, like the reference */
		float* cp = g->camera_planes + 6 * idx; float* rp = g->ray_planes + 2 * idx; float* nrm = g->normals + 3 * idx;
		{
			sig_inv si = sigma_inverse(cov6);
			m3 cci = m3_mul(m3_mul(m3_t(Wm), si.inv), Wm);
			v3 uvh = v3_make(txtz, tytz, 1), uvh_m = m3_mulv(cci, uvh), uvh_mn = v3_normalize(uvh_m);
			if (isnan(uvh_mn.v[0]) || !si.solved) {
				memset(cp, 0, 6 * sizeof(float)); rp[0] = rp[1] = 0; nrm[0] = nrm[1] = nrm[2] = 0;
			} else {
				float u2 = txtz * txtz, v2 = tytz * tytz, uv = txtz * tytz;
				float l = sqrtf(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
				m3 nJ = m3_make(1 / t[2], 0.0f, -(t[0]) / (t[2] * t[2]), 0.0f, 1 / t[2], -(t[1]) / (t[2] * t[2]), t[0] / l, t[1] / l, t[2] / l);
				m3 nJi = m3_make(v2 + 1, -uv, 0, -uv, u2 + 1, 0, -txtz, -tytz, 0);
				float vbn = v3_dot(uvh_mn, uvh);
				float fn = l / (u2 + v2 + 1);
				v3 plane = m3_mulv(nJi, v3_div(uvh_mn, fmaxf2(vbn, 0.0000001f)));
				float nl = u2 + v2 + 1;
				cp[0] = (-(v2 + 1) * t[2] + plane.v[0] * t[0]) / nl / focal_x; cp[1] = (uv * t[2] + plane.v[1] * t[0]) / nl / focal_y;
				cp[2] = (uv * t[2] + plane.v[0] * t[1]) / nl / focal_x; cp[3] = (-(u2 + 1) * t[2] + plane.v[1] * t[1]) / nl / focal_y;
				cp[4] = (t[0] + plane.v[0] * t[2]) / nl / focal_x; cp[5] = (t[1] + plane.v[1] * t[2]) / nl / focal_y;
				rp[0] = plane.v[0] * l / nl / focal_x; rp[1] = plane.v[1] * l / nl / focal_y;
				v3 rn = v3_make(-plane.v[0] * fn, -plane.v[1] * fn, -1);
				v3 n = v3_normalize(m3_mulv(nJ, rn));
				nrm[0] = n.v[0]; nrm[1] = n.v[1]; nrm[2] = n.v[2];
			}
		}
		g->ts[idx] = sqrtf(pv[0] * pv[0] + pv[1] * pv[1] + pv[2] * pv[2]);
		float det = cov2[0] * cov2[2] - cov2[1] * cov2[1];
		if (det == 0.0f) continue;
		float det_inv = 1.f / det;
		float conic[3] = {cov2[2] * det_inv, -cov2[1] * det_inv, cov2[0] * det_inv};
		float mid = 0.5f * (cov2[0] + cov2[2]);
		float lambda1 = mid + sqrtf(fmaxf2(0.1f, mid * mid - det));
		float lambda2 = mid - sqrtf(fmaxf2(0.1f, mid * mid - det));
		float my_radius = ceilf(3.f * sqrtf(fmaxf2(lambda1, lambda2)));
		float pix = ndc2pix(pp[0], s->W), piy = ndc2pix(pp[1], s->H);
		int x0, y0, x1, y1; get_rect(pix, piy, (int)my_radius, gx, gy, &x0, &y0, &x1, &y1);
		if ((x1 - x0) * (y1 - y0) == 0) continue;
		if (!s->colors_precomp) {
			/* forward.cu:23-74 */
			const float* cam = s->cam_pos;
			float dir[3] = {po[0] - cam[0], po[1] - cam[1], po[2] - cam[2]};
			float len = sqrtf(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
			float x = dir[0] / len, y = dir[1] / len, z = dir[2] / len;
			const float* sh = s->shs + (size_t)idx * s->M * 3;
			for (int ch = 0; ch < 3; ch++) {
#define SHC(k) sh[3 * (k) + ch]
				float res = SH_C0 * SHC(0);
				if (s->D > 0) {
					res = res - SH_C1 * y * SHC(1) + SH_C1 * z * SHC(2) - SH_C1 * x * SHC(3);
					if (s->D > 1) {
						float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
						res = res + SH_C2[0] * xy * SHC(4) + SH_C2[1] * yz * SHC(5) + SH_C2[2] * (2.0f * zz - xx - yy) * SHC(6) +
						      SH_C2[3] * xz * SHC(7) + SH_C2[4] * (xx - yy) * SHC(8);
						if (s->D > 2)
							res = res + SH_C3[0] * y * (3.0f * xx - yy) * SHC(9) + SH_C3[1] * xy * z * SHC(10) +
							      SH_C3[2] * y * (4.0f * zz - xx - yy) * SHC(11) + SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * SHC(12) +
							      SH_C3[4] * x * (4.0f * zz - xx - yy) * SHC(13) + SH_C3[5] * z * (xx - yy) * SHC(14) + SH_C3[6] * x * (xx - 3.0f * yy) * SHC(15);
					}
				}
#undef SHC
				res += 0.5f;
				g->clamped[3 * idx + ch] = res < 0;
				g->rgb[3 * idx + ch] = res < 0 ? 0.0f : res;
			}
		} else {
			for (int ch = 0; ch < 3; ch++) g->rgb[3 * idx + ch] = s->colors_precomp[3 * idx + ch];
		}
		g->depths[idx] = pv[2];
		memcpy(g->view_points + 3 * idx, pv, 3 * sizeof(float));
		g->radii[idx] = (int)my_radius;
		g->means2D[2 * idx] = pix; g->means2D[2 * idx + 1] = piy;
		g->conic_opacity[4 * idx] = conic[0]; g->conic_opacity[4 * idx + 1] = conic[1]; g->conic_opacity[4 * idx + 2] = conic[2];
		g->conic_opacity[4 * idx + 3] = s->opacities[idx] * coef;
		g->tiles_touched[idx] = (uint32_t)((y1 - y0) * (x1 - x0));
	}
}

/* ---- binning: rasterizer_impl.cu:70-111, 373-381, 151-173 ------------------------------------------------- */
typedef struct { uint64_t key; uint32_t val; } kv;
static void merge_sort(kv* a, kv* tmp, size_t n) {  /* stable */
	if (n < 2) return;
	size_t h = n / 2;
	merge_sort(a, tmp, h); merge_sort(a + h, tmp, n - h);
	size_t i = 0, j = h, k = 0;
	while (i < h && j < n) tmp[k++] = (a[j].key < a[i].key) ? a[j++] : a[i++];
	while (i < h) tmp[k++] = a[i++];
	while (j < n) tmp[k++] = a[j++];
	memcpy(a, tmp, n * sizeof(kv));
}
/* returns num_rendered; keys/vals sized by the caller from sum(tiles_touched); ranges[tiles][2] */
int64_t orc_binning(int P, int W, int H, const int* radii, const float* means2D, const float* depths, uint64_t* keys, uint32_t* vals, uint32_t* ranges) {
	const int gx = (W + TILE - 1) / TILE, gy = (H + TILE - 1) / TILE;
	size_t n = 0;
	for (int idx = 0; idx < P; idx++) {
		if (radii[idx] <= 0) continue;
		int x0, y0, x1, y1; get_rect(means2D[2 * idx], means2D[2 * idx + 1], radii[idx], gx, gy, &x0, &y0, &x1, &y1);
		uint32_t dbits; memcpy(&dbits, depths + idx, 4);
		for (int y = y0; y < y1; y++) for (int x = x0; x < x1; x++) { keys[n] = ((uint64_t)(y * gx + x) << 32) | dbits; vals[n] = (uint32_t)idx; n++; }
	}
	kv* a = (kv*)malloc((n + 1) * sizeof(kv)); kv* tmp = (kv*)malloc((n + 1) * sizeof(kv));
	for (size_t i = 0; i < n; i++) { a[i].key = keys[i]; a[i].val = vals[i]; }
	merge_sort(a, tmp, n);
	for (size_t i = 0; i < n; i++) { keys[i] = a[i].key; vals[i] = a[i].val; }
	free(a); free(tmp);
	memset(ranges, 0, (size_t)gx * gy * 2 * sizeof(uint32_t));
	for (size_t i = 0; i < n; i++) {
		uint32_t cur = (uint32_t)(keys[i] >> 32);
		if (i == 0) ranges[2 * cur] = 0;
		else { uint32_t prev = (uint32_t)(keys[i - 1] >> 32); if (cur != prev) { ranges[2 * prev + 1] = (uint32_t)i; ranges[2 * cur] = (uint32_t)i; } }
		if (i == n - 1) ranges[2 * cur + 1] = (uint32_t)n;
	}
	return (int64_t)n;
}

/* ---- forward blend: forward.cu:428-693 ---------------------------------------------------------------------- */
typedef struct {
	float *color, *coord, *mcoord, *alpha, *normal, *depth, *mdepth;   /* API maps, CHW */
	uint32_t* n_contrib;                                                 /* [2,H,W] */
	float *accum_coord, *accum_depth, *normal_length;
} orc_image;

void orc_render_forward(int W, int H, float tan_fovx, float tan_fovy, const float* bg, int require_coord, int require_depth,
                        const uint32_t* ranges, const uint32_t* point_list, const orc_geom* g, orc_image* o) {
	const int gx = (W + TILE - 1) / TILE;
	const float focal_y = H / (2.0f * tan_fovy), focal_x = W / (2.0f * tan_fovx);
	const int COORD = require_coord, DEPTH = require_depth, NORMAL = require_coord || require_depth, GEO = NORMAL;
	const size_t HW = (size_t)H * W;
	for (int py = 0; py < H; py++) for (int px = 0; px < W; px++) {
		const size_t pix = (size_t)W * py + px;
		const float pxf = (float)px, pyf = (float)py;
		const float pnx = (pxf - W / 2.f) / focal_x, pny = (pyf - H / 2.f) / focal_y;
		const float ln = sqrtf(pnx * pnx + pny * pny + 1);
		const uint32_t* rg = ranges + 2 * ((py / TILE) * gx + px / TILE);
		float T = 1.0f, C[3] = {0, 0, 0}, weight = 0, Coord[3] = {0, 0, 0}, mCoord[3] = {0, 0, 0}, Depth = 0, mDepth = 0, Normal[3] = {0, 0, 0};
		uint32_t contributor = 0, last = 0, maxc = 0xFFFFFFFFu;
		for (uint32_t it = rg[0]; it < rg[1]; it++) {
			contributor++;
			const int id = (int)point_list[it];
			const float dx = g->means2D[2 * id] - pxf, dy = g->means2D[2 * id + 1] - pyf;
			const float* co = g->conic_opacity + 4 * id;
			const float power = -0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
			if (power > 0.0f) continue;
			const float alpha = fminf2(0.99f, co[3] * expf(power));
			if (alpha < 1.0f / 255.0f) continue;
			const float test_T = T * (1 - alpha);
			if (test_T < 0.0001f) break;   /* done: nothing after this can change the pixel */
			const float aT = alpha * T;
			for (int ch = 0; ch < 3; ch++) C[ch] += g->rgb[3 * id + ch] * aT;
			const int before_median = T > 0.5;
			if (COORD) {
				const float* cpl = g->camera_planes + 6 * id; const float* vp = g->view_points + 3 * id;
				for (int ch = 0; ch < 3; ch++) {
					const float c = vp[ch] + cpl[2 * ch] * dx + cpl[2 * ch + 1] * dy;
					Coord[ch] += c * aT; if (before_median) mCoord[ch] = c;
				}
			}
			if (DEPTH) {
				const float t = g->ts[id] + (g->ray_planes[2 * id] * dx + g->ray_planes[2 * id + 1] * dy);
				Depth += t * aT; if (before_median) mDepth = t;
			}
			if (NORMAL) for (int ch = 0; ch < 3; ch++) Normal[ch] += g->normals[3 * id + ch] * aT;
			if (GEO && before_median) maxc = contributor;
			weight += aT; T = test_T; last = contributor;
		}
		o->n_contrib[pix] = last; o->n_contrib[pix + HW] = maxc;
		for (int ch = 0; ch < 3; ch++) o->color[ch * HW + pix] = C[ch] + T * bg[ch];
		o->alpha[pix] = weight;
		if (COORD) for (int ch = 0; ch < 3; ch++) {
			o->coord[ch * HW + pix] = last ? Coord[ch] / weight : 0; o->accum_coord[ch * HW + pix] = Coord[ch]; o->mcoord[ch * HW + pix] = mCoord[ch];
		}
		if (DEPTH) {
			const float dln = Depth / ln;
			o->accum_depth[pix] = dln; o->depth[pix] = last ? dln / weight : 0; o->mdepth[pix] = mDepth / ln;
		}
		if (NORMAL) {
			if (last) {
				float len = sqrtf(Normal[0] * Normal[0] + Normal[1] * Normal[1] + Normal[2] * Normal[2]);
				o->normal_length[pix] = len; len = fmaxf2(len, 1.0E-12F);
				for (int ch = 0; ch < 3; ch++) o->normal[ch * HW + pix] = Normal[ch] / len;
			} else { o->normal_length[pix] = 1; for (int ch = 0; ch < 3; ch++) o->normal[ch * HW + pix] = 0; }
		}
	}
}

/* ---- backward blend: backward.cu:631-1016.  Intermediate per-Gaussian gradients, summed in double. -------- */
typedef struct {
	double *mean2D /*[P,3]*/, *conic /*[P,4]*/, *opacity /*[P]*/, *colors /*[P,3]*/, *ts /*[P]*/, *camera_planes /*[P,6]*/, *ray_planes /*[P,2]*/,
	    *normals /*[P,3]*/, *view_points /*[P,3]*/;
} orc_sgrad;
typedef struct { const float *color, *coord, *mcoord, *depth, *mdepth, *alpha, *normal; } orc_upstream;

void orc_render_backward(int W, int H, float tan_fovx, float tan_fovy, const float* bg, int require_coord, int require_depth,
                         const uint32_t* ranges, const uint32_t* point_list, const orc_geom* g, const orc_image* f, const orc_upstream* u, orc_sgrad* sg) {
	const int gx = (W + TILE - 1) / TILE;
	const float focal_y = H / (2.0f * tan_fovy), focal_x = W / (2.0f * tan_fovx);
	const int COORD = require_coord, DEPTH = require_depth, NORMAL = require_coord || require_depth, GEO = NORMAL;
	const size_t HW = (size_t)H * W;
	const float ddelx_dx = (float)(0.5 * W), ddely_dy = (float)(0.5 * H);
	for (int py = 0; py < H; py++) for (int px = 0; px < W; px++) {
		const size_t pix = (size_t)W * py + px;
		const float pxf = (float)px, pyf = (float)py;
		const float pnx = (pxf - W / 2.f) / focal_x, pny = (pyf - H / 2.f) / focal_y;
		const float ln = sqrtf(pnx * pnx + pny * pny + 1);
		const uint32_t* rg = ranges + 2 * ((py / TILE) * gx + px / TILE);
		const float T_final = 1 - f->alpha[pix], w_final = f->alpha[pix];
		float T = T_final;
		const int last_contributor = (int)f->n_contrib[pix], max_contributor = (int)f->n_contrib[pix + HW];
		float dL_dpixel[3], dL_dalpha = u->alpha[pix], dpc[3] = {0, 0, 0}, dpmc[3] = {0, 0, 0}, dpt = 0, dpmt = 0, dpn[3] = {0, 0, 0};
		for (int i = 0; i < 3; i++) dL_dpixel[i] = u->color[i * HW + pix];
		if (GEO) {
			const float ww = w_final * w_final;
			if (COORD) for (int i = 0; i < 3; i++) {
				const float gw = u->coord[i * HW + pix];
				dL_dalpha -= gw * f->accum_coord[i * HW + pix] / ww; dpc[i] = gw / w_final; dpmc[i] = u->mcoord[i * HW + pix];
			}
			if (DEPTH) {
				const float gw = u->depth[pix];
				dL_dalpha -= gw * f->accum_depth[pix] / ww; dpt = gw / w_final / ln; dpmt = u->mdepth[pix] / ln;
			}
			if (NORMAL) {
				const float gn[3] = {u->normal[pix], u->normal[HW + pix], u->normal[2 * HW + pix]};
				const float nn[3] = {f->normal[pix], f->normal[HW + pix], f->normal[2 * HW + pix]};
				const float nlen = f->normal_length[pix];
				if (nlen < 1.0E-12F) for (int i = 0; i < 3; i++) dpn[i] = gn[i] / 1.0E-12F;
				else {
					float t0 = gn[0] * nn[0], t1 = gn[1] * nn[1], t2 = gn[2] * nn[2];
					float d = t0 + t1 + t2;
					for (int i = 0; i < 3; i++) dpn[i] = (gn[i] - d * nn[i]) / nlen;
				}
			}
		}
		float accum_rec[3] = {0, 0, 0}, last_color[3] = {0, 0, 0}, accum_coord_rec[3] = {0, 0, 0}, last_coord[3] = {0, 0, 0};
		float accum_t_rec = 0, last_t = 0, accum_normal_rec[3] = {0, 0, 0}, last_normal[3] = {0, 0, 0}, accum_alpha_rec = 0, last_alpha = 0;
		float bg_dot = 0; for (int i = 0; i < 3; i++) bg_dot += bg[i] * dL_dpixel[i];
		for (int64_t it = (int64_t)rg[1] - 1; it >= (int64_t)rg[0]; it--) {
			const int contributor = (int)(it - rg[0]);
			if (contributor >= last_contributor) continue;
			const int id = (int)point_list[it];
			const float dx = g->means2D[2 * id] - pxf, dy = g->means2D[2 * id + 1] - pyf;
			const float* co = g->conic_opacity + 4 * id;
			const float power = -0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
			if (power > 0.0f) continue;
			const float G = expf(power);
			const float alpha = fminf2(0.99f, co[3] * G);
			if (alpha < 1.0f / 255.0f) continue;
			T = T / (1.f - alpha);
			const float dch = alpha * T;
			float dL_dopa = 0.0f;
			for (int ch = 0; ch < 3; ch++) {
				const float c = g->rgb[3 * id + ch];
				accum_rec[ch] = last_alpha * last_color[ch] + (1.f - last_alpha) * accum_rec[ch]; last_color[ch] = c;
				dL_dopa += (c - accum_rec[ch]) * dL_dpixel[ch];
				sg->colors[3 * id + ch] += dch * dL_dpixel[ch];
			}
			float dcoords[3] = {0, 0, 0}, dL_dt = 0;
			const float* cpl = g->camera_planes + 6 * id; const float* rpl = g->ray_planes + 2 * id;
			if (COORD) {
				const float* vp = g->view_points + 3 * id;
				for (int ch = 0; ch < 3; ch++) {
					const float c = vp[ch] + cpl[2 * ch] * dx + cpl[2 * ch + 1] * dy;
					accum_coord_rec[ch] = last_alpha * last_coord[ch] + (1.f - last_alpha) * accum_coord_rec[ch]; last_coord[ch] = c;
					dL_dopa += (c - accum_coord_rec[ch]) * dpc[ch];
					dcoords[ch] = dch * dpc[ch];
					if (contributor == max_contributor - 1) dcoords[ch] += dpmc[ch];
					sg->view_points[3 * id + ch] += dcoords[ch];
					sg->camera_planes[6 * id + 2 * ch] += dcoords[ch] * dx / focal_x;
					sg->camera_planes[6 * id + 2 * ch + 1] += dcoords[ch] * dy / focal_y;
				}
			}
			if (DEPTH) {
				const float t = g->ts[id] + (rpl[0] * dx + rpl[1] * dy);
				accum_t_rec = last_alpha * last_t + (1.f - last_alpha) * accum_t_rec; last_t = t;
				dL_dopa += (t - accum_t_rec) * dpt;
				dL_dt = dch * dpt;
				if (contributor == max_contributor - 1) dL_dt += dpmt;
				sg->ts[id] += dL_dt; sg->ray_planes[2 * id] += dL_dt * dx / focal_x; sg->ray_planes[2 * id + 1] += dL_dt * dy / focal_y;
			}
			if (NORMAL) for (int ch = 0; ch < 3; ch++) {
				const float c = g->normals[3 * id + ch];
				accum_normal_rec[ch] = last_alpha * last_normal[ch] + (1.f - last_alpha) * accum_normal_rec[ch]; last_normal[ch] = c;
				dL_dopa += (c - accum_normal_rec[ch]) * dpn[ch];
				sg->normals[3 * id + ch] += dch * dpn[ch];
			}
			accum_alpha_rec = last_alpha + (1.f - last_alpha) * accum_alpha_rec;
			dL_dopa += (1 - accum_alpha_rec) * dL_dalpha;
			dL_dopa *= T;
			last_alpha = alpha;
			dL_dopa += (-T_final / (1.f - alpha)) * bg_dot;
			const float dL_dG = co[3] * dL_dopa;
			const float gdx = G * dx, gdy = G * dy;
			const float dG_ddelx = -gdx * co[0] - gdy * co[1], dG_ddely = -gdy * co[2] - gdx * co[1];
			float dL_ddelx = dL_dG * dG_ddelx, dL_ddely = dL_dG * dG_ddely;
			if (COORD) {
				dL_ddelx += dcoords[0] * cpl[0] + dcoords[1] * cpl[2] + dcoords[2] * cpl[4];
				dL_ddely += dcoords[0] * cpl[1] + dcoords[1] * cpl[3] + dcoords[2] * cpl[5];
			}
			if (DEPTH) { dL_ddelx += dL_dt * rpl[0]; dL_ddely += dL_dt * rpl[1]; }
			sg->mean2D[3 * id] += dL_ddelx * ddelx_dx; sg->mean2D[3 * id + 1] += dL_ddely * ddely_dy;
			sg->mean2D[3 * id + 2] += fabsf(dL_dG * dG_ddelx * ddelx_dx) + fabsf(dL_dG * dG_ddely * ddely_dy);
			sg->conic[4 * id] += -0.5f * gdx * dx * dL_dG; sg->conic[4 * id + 1] += -0.5f * gdx * dy * dL_dG; sg->conic[4 * id + 3] += -0.5f * gdy * dy * dL_dG;
			sg->opacity[id] += G * dL_dopa;
		}
	}
}

/* ---- backward preprocess: backward.cu:145-488 then :560-628 ------------------------------------------------ */
typedef struct { float *means2D, *colors, *opacity, *means3D, *cov3D, *sh, *scales, *rotations; } orc_pgrad;

void orc_preprocess_backward(const orc_scene* s, const orc_geom* g, const orc_sgrad* sg, orc_pgrad* o, int fix_mip_gradient) {
	const float h_y = s->H / (2.0f * s->tan_fovy), h_x = s->W / (2.0f * s->tan_fovx);
	const float* V = s->viewmatrix; const float ks = s->kernel_size; const int M = s->M;
	for (int idx = 0; idx < s->P; idx++) {
		/* what the API returns straight from the scatter stage */
		for (int i = 0; i < 3; i++) { o->means2D[3 * idx + i] = (float)sg->mean2D[3 * idx + i]; o->colors[3 * idx + i] = (float)sg->colors[3 * idx + i]; }
		o->opacity[idx] = (float)sg->opacity[idx];
		if (!(g->radii[idx] > 0)) continue;
		const float* cov3D = s->cov3D_precomp ? s->cov3D_precomp + 6 * idx : g->cov3D + 6 * idx;
		const float* mean = s->means3D + 3 * idx;
		const float dcon[3] = {(float)sg->conic[4 * idx], (float)sg->conic[4 * idx + 1], (float)sg->conic[4 * idx + 3]};
		v3 dL_dnormal = v3_make((float)sg->normals[3 * idx], (float)sg->normals[3 * idx + 1], (float)sg->normals[3 * idx + 2]);
		/* rasterizer_impl.cu:569 hands dL_dconic where conic_opacity is expected: `.w` is dL/dconic_yy */
		const float combined_opacity = fix_mip_gradient ? g->conic_opacity[4 * idx + 3] : (float)sg->conic[4 * idx + 3];
		const float d0x = (float)sg->camera_planes[6 * idx], d0y = (float)sg->camera_planes[6 * idx + 1];
		const float d1x = (float)sg->camera_planes[6 * idx + 2], d1y = (float)sg->camera_planes[6 * idx + 3];
		const float d2x = (float)sg->camera_planes[6 * idx + 4], d2y = (float)sg->camera_planes[6 * idx + 5];
		const float drx = (float)sg->ray_planes[2 * idx], dry = (float)sg->ray_planes[2 * idx + 1];
		float t[3]; xf4x3(mean, V, t);
		const float limx = 1.3f * s->tan_fovx, limy = 1.3f * s->tan_fovy;
		float txtz = t[0] / t[2], tytz = t[1] / t[2];
		t[0] = fminf2(limx, fmaxf2(-limx, txtz)) * t[2]; t[1] = fminf2(limy, fmaxf2(-limy, tytz)) * t[2];
		const float xgm = (txtz < -limx || txtz > limx) ? 0 : 1, ygm = (tytz < -limy || tytz > limy) ? 0 : 1;
		txtz = t[0] / t[2]; tytz = t[1] / t[2];
		m3 J = m3_make(h_x / t[2], 0.0f, -(h_x * t[0]) / (t[2] * t[2]), 0.0f, h_y / t[2], -(h_y * t[1]) / (t[2] * t[2]), 0, 0, 0);
		m3 Wm = m3_make(V[0], V[4], V[8], V[1], V[5], V[9], V[2], V[6], V[10]);
		m3 Vrk = m3_make(cov3D[0], cov3D[1], cov3D[2], cov3D[1], cov3D[3], cov3D[4], cov3D[2], cov3D[4], cov3D[5]);
		m3 T = m3_mul(Wm, J);
		m3 c2 = m3_mul(m3_mul(m3_t(T), m3_t(Vrk)), T);
		const float det_0 = (float)fmax(1e-6, (double)(c2.c[0][0] * c2.c[1][1] - c2.c[0][1] * c2.c[0][1]));
		const float det_1 = (float)fmax(1e-6, (double)((c2.c[0][0] + ks) * (c2.c[1][1] + ks) - c2.c[0][1] * c2.c[0][1]));
		const float coef = (float)sqrt(det_0 / (det_1 + 1e-6) + 1e-6);
		sig_inv si = sigma_inverse(cov3D);
		m3 cci = m3_mul(m3_mul(m3_t(Wm), si.inv), Wm);
		v3 uvh = v3_make(txtz, tytz, 1), uvh_m = m3_mulv(cci, uvh), uvh_mn = v3_normalize(uvh_m);
		const float u2 = txtz * txtz, v2 = tytz * tytz, uv = txtz * tytz;
		m3 dVrk = m3_zero(), dnJ = m3_zero();
		float plane[3] = {0, 0, 0}, dL_du = 0, dL_dv = 0, dL_dl = 0, l = 1, nl = 1;
		if (!(isnan(uvh_mn.v[0]) || !si.solved)) {
			const float vb = v3_dot(uvh_m, uvh), vbn = v3_dot(uvh_mn, uvh);
			l = sqrtf(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
			m3 nJ = m3_make(1 / t[2], 0.0f, -(t[0]) / (t[2] * t[2]), 0.0f, 1 / t[2], -(t[1]) / (t[2] * t[2]), t[0] / l, t[1] / l, t[2] / l);
			m3 nJi = m3_make(v2 + 1, -uv, 0, -uv, u2 + 1, 0, -txtz, -tytz, 0);
			const float cvb = fmaxf2(vb, 0.0000001f), cvbn = fmaxf2(vbn, 0.0000001f);
			nl = u2 + v2 + 1;
			const float fn = l / nl;
			v3 q = v3_div(uvh_mn, cvbn);
			v3 pl = m3_mulv(nJi, q); plane[0] = pl.v[0]; plane[1] = pl.v[1]; plane[2] = pl.v[2];
			const float c0x = (-(v2 + 1) * t[2] + plane[0] * t[0]) / nl, c0y = (uv * t[2] + plane[1] * t[0]) / nl;
			const float c1x = (uv * t[2] + plane[0] * t[1]) / nl, c1y = (-(u2 + 1) * t[2] + plane[1] * t[1]) / nl;
			const float c2x = (t[0] + plane[0] * t[2]) / nl, c2y = (t[1] + plane[1] * t[2]) / nl;
			const float rpx = plane[0] * fn, rpy = plane[1] * fn;
			v3 rn = v3_make(-plane[0] * fn, -plane[1] * fn, -1);
			v3 cn = m3_mulv(nJ, rn), nvec = v3_normalize(cn);
			const float lv = sqrtf(v3_dot(cn, cn));
			v3 dn_lv = v3_div(dL_dnormal, lv);
			v3 dcn = v3_sub(dn_lv, v3_scale(nvec, v3_dot(nvec, dn_lv)));
			v3 drn = m3_mulv(m3_t(nJ), dcn);
			dnJ = m3_outer(dcn, rn);
			dL_dl = (-plane[0] * drn.v[0] - plane[1] * drn.v[1] + plane[0] * drx + plane[1] * dry) / nl;
			const float dpx = (t[0] * d0x + t[1] * d1x + t[2] * d2x - l * drn.v[0] + drx * l) / nl;
			const float dpy = (t[0] * d0y + t[1] * d1y + t[2] * d2y - l * drn.v[1] + dry * l) / nl;
			v3 dp3 = v3_make(dpx, dpy, 0);
			const float dL_dnl = (-d0x * c0x - d0y * c0y - d1x * c1x - d1y * c1y - d2x * c2x - d2y * c2y - drn.v[0] * rn.v[0] - drn.v[1] * rn.v[1] -
			                      drx * rpx - dry * rpy) / nl;
			const float tmp = dpx * plane[0] + dpy * plane[1];
			v3 W_uvh = m3_mulv(Wm, uvh);
			if (si.well) {
				v3 rhs = v3_add(v3_scale(W_uvh, -tmp), m3_mulv(m3_mul(Wm, m3_t(nJi)), dp3));
				dVrk = m3_scale(m3_outer(m3_mulv(si.inv, W_uvh), m3_mulv(m3_div(si.inv, cvb), rhs)), -1.0f);
			} else {
				const float dL_dvb = -tmp / cvb;
				v3 nji = m3_mulv(m3_t(nJi), v3_make(dpx / cvb, dpy / cvb, 0));
				m3 dVi = m3_outer(W_uvh, v3_add(v3_scale(W_uvh, dL_dvb), m3_mulv(Wm, nji)));
				v3 emin = v3_make(si.E.c[si.min_id][0], si.E.c[si.min_id][1], si.E.c[si.min_id][2]);
				v3 dLdv = m3_mulv(m3_add(dVi, m3_t(dVi)), emin);
				for (int j = 0; j < 3; j++) if (j != si.min_id) {
					v3 ej = v3_make(si.E.c[j][0], si.E.c[j][1], si.E.c[j][2]);
					const float sc = v3_dot(ej, dLdv) / fminf2(si.lam[si.min_id] - si.lam[j], -0.0000001f);
					dVrk = m3_add(dVrk, m3_outer(v3_scale(ej, sc), emin));
				}
			}
			v3 duvh = v3_add(v3_scale(q, 2 * (-tmp)), m3_mulv(m3_mul(m3_div(cci, cvb), m3_t(nJi)), dp3));
			m3 dnJi = m3_outer(dp3, q);
			dL_du = dL_dnl * 2 * txtz + duvh.v[0] + (dnJi.c[0][1] + dnJi.c[1][0]) * (-tytz) + 2 * dnJi.c[1][1] * txtz - dnJi.c[2][0] +
			        (d0y * t[1] + d1x * t[1] + d1y * (-2 * t[0])) / nl;
			dL_dv = dL_dnl * 2 * tytz + duvh.v[1] + (dnJi.c[0][1] + dnJi.c[1][0]) * (-txtz) + 2 * dnJi.c[0][0] * tytz - dnJi.c[2][1] +
			        (d0x * (-2 * t[1]) + d0y * t[0] + d1x * t[0]) / nl;
		}
		/* backward.cu:367-431 */
		float dL_dopacity = (float)sg->opacity[idx];
		const float opacity = (float)(combined_opacity / (coef + 1e-6));
		const float dL_dcoef = dL_dopacity * opacity;
		const float dL_dsqrtcoef = (float)(dL_dcoef * 0.5 * 1. / (coef + 1e-6));
		const float dL_ddet0 = (float)(dL_dsqrtcoef / (det_1 + 1e-6));
		const float dL_ddet1 = (float)(dL_dsqrtcoef * det_0 * (-1.f / (det_1 * det_1 + 1e-6)));
		const float dcoef_da = dL_ddet0 * c2.c[1][1] + dL_ddet1 * (c2.c[1][1] + ks);
		const float dcoef_db = (float)(dL_ddet0 * (-2. * c2.c[0][1]) + dL_ddet1 * (-2. * c2.c[0][1]));
		const float dcoef_dc = dL_ddet0 * c2.c[0][0] + dL_ddet1 * (c2.c[0][0] + ks);
		const float a = c2.c[0][0] + ks, b = c2.c[0][1], c = c2.c[1][1] + ks;
		const float denom = a * c - b * b;
		float dL_da = 0, dL_db = 0, dL_dc = 0;
		const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
		float* dcov = o->cov3D + 6 * idx;
#define TT(cc, rr) T.c[cc][rr]
#define VV(cc, rr) Vrk.c[cc][rr]
		if (denom2inv != 0) {
			dL_da = denom2inv * (-c * c * dcon[0] + 2 * b * c * dcon[1] + (denom - a * c) * dcon[2]);
			dL_dc = denom2inv * (-a * a * dcon[2] + 2 * a * b * dcon[1] + (denom - a * c) * dcon[0]);
			dL_db = denom2inv * 2 * (b * c * dcon[0] - (denom + 2 * b * b) * dcon[1] + a * b * dcon[2]);
			if (det_0 <= 1e-6 || det_1 <= 1e-6) dL_dopacity = 0;
			else { dL_da += dcoef_da; dL_dc += dcoef_dc; dL_db += dcoef_db; dL_dopacity = dL_dopacity * coef; }
			dcov[0] = (TT(0, 0) * TT(0, 0) * dL_da + TT(0, 0) * TT(1, 0) * dL_db + TT(1, 0) * TT(1, 0) * dL_dc);
			dcov[3] = (TT(0, 1) * TT(0, 1) * dL_da + TT(0, 1) * TT(1, 1) * dL_db + TT(1, 1) * TT(1, 1) * dL_dc);
			dcov[5] = (TT(0, 2) * TT(0, 2) * dL_da + TT(0, 2) * TT(1, 2) * dL_db + TT(1, 2) * TT(1, 2) * dL_dc);
			dcov[1] = 2 * TT(0, 0) * TT(0, 1) * dL_da + (TT(0, 0) * TT(1, 1) + TT(0, 1) * TT(1, 0)) * dL_db + 2 * TT(1, 0) * TT(1, 1) * dL_dc;
			dcov[2] = 2 * TT(0, 0) * TT(0, 2) * dL_da + (TT(0, 0) * TT(1, 2) + TT(0, 2) * TT(1, 0)) * dL_db + 2 * TT(1, 0) * TT(1, 2) * dL_dc;
			dcov[4] = 2 * TT(0, 2) * TT(0, 1) * dL_da + (TT(0, 1) * TT(1, 2) + TT(0, 2) * TT(1, 1)) * dL_db + 2 * TT(1, 1) * TT(1, 2) * dL_dc;
		} else for (int i = 0; i < 6; i++) dcov[i] = 0;
		o->opacity[idx] = dL_dopacity;
		dcov[0] += dVrk.c[0][0]; dcov[3] += dVrk.c[1][1]; dcov[5] += dVrk.c[2][2];
		dcov[1] += dVrk.c[0][1] + dVrk.c[1][0]; dcov[2] += dVrk.c[0][2] + dVrk.c[2][0]; dcov[4] += dVrk.c[1][2] + dVrk.c[2][1];
		const float dT00 = 2 * (TT(0, 0) * VV(0, 0) + TT(0, 1) * VV(0, 1) + TT(0, 2) * VV(0, 2)) * dL_da + (TT(1, 0) * VV(0, 0) + TT(1, 1) * VV(0, 1) + TT(1, 2) * VV(0, 2)) * dL_db;
		const float dT01 = 2 * (TT(0, 0) * VV(1, 0) + TT(0, 1) * VV(1, 1) + TT(0, 2) * VV(1, 2)) * dL_da + (TT(1, 0) * VV(1, 0) + TT(1, 1) * VV(1, 1) + TT(1, 2) * VV(1, 2)) * dL_db;
		const float dT02 = 2 * (TT(0, 0) * VV(2, 0) + TT(0, 1) * VV(2, 1) + TT(0, 2) * VV(2, 2)) * dL_da + (TT(1, 0) * VV(2, 0) + TT(1, 1) * VV(2, 1) + TT(1, 2) * VV(2, 2)) * dL_db;
		const float dT10 = 2 * (TT(1, 0) * VV(0, 0) + TT(1, 1) * VV(0, 1) + TT(1, 2) * VV(0, 2)) * dL_dc + (TT(0, 0) * VV(0, 0) + TT(0, 1) * VV(0, 1) + TT(0, 2) * VV(0, 2)) * dL_db;
		const float dT11 = 2 * (TT(1, 0) * VV(1, 0) + TT(1, 1) * VV(1, 1) + TT(1, 2) * VV(1, 2)) * dL_dc + (TT(0, 0) * VV(1, 0) + TT(0, 1) * VV(1, 1) + TT(0, 2) * VV(1, 2)) * dL_db;
		const float dT12 = 2 * (TT(1, 0) * VV(2, 0) + TT(1, 1) * VV(2, 1) + TT(1, 2) * VV(2, 2)) * dL_dc + (TT(0, 0) * VV(2, 0) + TT(0, 1) * VV(2, 1) + TT(0, 2) * VV(2, 2)) * dL_db;
#undef TT
#undef VV
		const float dJ00 = Wm.c[0][0] * dT00 + Wm.c[0][1] * dT01 + Wm.c[0][2] * dT02;
		const float dJ02 = Wm.c[2][0] * dT00 + Wm.c[2][1] * dT01 + Wm.c[2][2] * dT02;
		const float dJ11 = Wm.c[1][0] * dT10 + Wm.c[1][1] * dT11 + Wm.c[1][2] * dT12;
		const float dJ12 = Wm.c[2][0] * dT10 + Wm.c[2][1] * dT11 + Wm.c[2][2] * dT12;
		const float tz = 1.f / t[2], tz2 = tz * tz, tz3 = tz2 * tz, l3 = l * l * l;
		const float dtx = xgm * (-h_x * tz2 * dJ02 + dL_du * tz - dnJ.c[0][2] * tz2 + dnJ.c[2][0] * (1 / l - t[0] * t[0] / l3) + dnJ.c[2][1] * (-t[0] * t[1] / l3) +
		                         dnJ.c[2][2] * (-t[0] * t[2] / l3) + (d0x * plane[0] + d0y * plane[1] + d2x) / nl + dL_dl * t[0] / l);
		const float dty = ygm * (-h_y * tz2 * dJ12 + dL_dv * tz - dnJ.c[1][2] * tz2 + dnJ.c[2][0] * (-t[0] * t[1] / l3) + dnJ.c[2][1] * (1 / l - t[1] * t[1] / l3) +
		                         dnJ.c[2][2] * (-t[1] * t[2] / l3) + (d1x * plane[0] + d1y * plane[1] + d2y) / nl + dL_dl * t[1] / l);
		const float dtz = -h_x * tz2 * dJ00 - h_y * tz2 * dJ11 + (2 * h_x * t[0]) * tz3 * dJ02 + (2 * h_y * t[1]) * tz3 * dJ12 - (dL_du * t[0] + dL_dv * t[1]) * tz2 +
		                  (dnJ.c[0][0] + dnJ.c[1][1]) * (-tz2) + dnJ.c[0][2] * (2 * t[0] * tz3) + dnJ.c[1][2] * (2 * t[1] * tz3) +
		                  (dnJ.c[2][0] * t[0] + dnJ.c[2][1] * t[1]) * (-t[2] / l3) + dnJ.c[2][2] * (1 / l - t[2] * t[2] / l3) +
		                  (d0x * (-(v2 + 1)) + d0y * uv + d1x * uv + d1y * (-(u2 + 1)) + d2x * plane[0] + d2y * plane[1]) / nl + dL_dl * t[2] / l;
		float dt3[3] = {dtx, dty, dtz}, dmean[3];
		xfvec4x3T(dt3, V, dmean);

		/* backward.cu:587-619 */
		{
			const float* proj = s->projmatrix;
			float mh[4]; xf4x4(mean, proj, mh);
			const float m_w = 1.0f / (mh[3] + 0.0000001f);
			const float mul1 = (proj[0] * mean[0] + proj[4] * mean[1] + proj[8] * mean[2] + proj[12]) * m_w * m_w;
			const float mul2 = (proj[1] * mean[0] + proj[5] * mean[1] + proj[9] * mean[2] + proj[13]) * m_w * m_w;
			const float gx2 = (float)sg->mean2D[3 * idx], gy2 = (float)sg->mean2D[3 * idx + 1];
			const float a1x = (proj[0] * m_w - proj[3] * mul1) * gx2 + (proj[1] * m_w - proj[3] * mul2) * gy2;
			const float a1y = (proj[4] * m_w - proj[7] * mul1) * gx2 + (proj[5] * m_w - proj[7] * mul2) * gy2;
			const float a1z = (proj[8] * m_w - proj[11] * mul1) * gx2 + (proj[9] * m_w - proj[11] * mul2) * gy2;
			float mv[3]; xf4x3(mean, V, mv);
			const float tl = sqrtf(mv[0] * mv[0] + mv[1] * mv[1] + mv[2] * mv[2]);
			const float dts = (float)sg->ts[idx];
			float in3[3] = {(float)sg->view_points[3 * idx] + mv[0] / tl * dts, (float)sg->view_points[3 * idx + 1] + mv[1] / tl * dts,
			                (float)sg->view_points[3 * idx + 2] + mv[2] / tl * dts}, a2[3];
			xfvec4x3T(in3, V, a2);
			dmean[0] += a1x + a2[0]; dmean[1] += a1y + a2[1]; dmean[2] += a1z + a2[2];
		}
		/* backward.cu:21-140 */
		if (s->shs) {
			const float* cam = s->cam_pos;
			const float dor[3] = {mean[0] - cam[0], mean[1] - cam[1], mean[2] - cam[2]};
			const float len = sqrtf(dor[0] * dor[0] + dor[1] * dor[1] + dor[2] * dor[2]);
			const float x = dor[0] / len, y = dor[1] / len, z = dor[2] / len;
			const float* sh = s->shs + (size_t)idx * M * 3; float* dsh = o->sh + (size_t)idx * M * 3;
			float dRGB[3]; for (int ch = 0; ch < 3; ch++) dRGB[ch] = o->colors[3 * idx + ch] * (g->clamped[3 * idx + ch] ? 0 : 1);
			float dx3[3] = {0, 0, 0}, dy3[3] = {0, 0, 0}, dz3[3] = {0, 0, 0};
#define SET(k, w) for (int ch = 0; ch < 3; ch++) dsh[3 * (k) + ch] = (w) * dRGB[ch]
#define S(k) sh[3 * (k) + ch]
			SET(0, SH_C0);
			if (s->D > 0) {
				SET(1, -SH_C1 * y); SET(2, SH_C1 * z); SET(3, -SH_C1 * x);
				for (int ch = 0; ch < 3; ch++) { dx3[ch] = -SH_C1 * S(3); dy3[ch] = -SH_C1 * S(1); dz3[ch] = SH_C1 * S(2); }
				if (s->D > 1) {
					const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
					SET(4, SH_C2[0] * xy); SET(5, SH_C2[1] * yz); SET(6, SH_C2[2] * (2.f * zz - xx - yy)); SET(7, SH_C2[3] * xz); SET(8, SH_C2[4] * (xx - yy));
					for (int ch = 0; ch < 3; ch++) {
						dx3[ch] += SH_C2[0] * y * S(4) + SH_C2[2] * 2.f * -x * S(6) + SH_C2[3] * z * S(7) + SH_C2[4] * 2.f * x * S(8);
						dy3[ch] += SH_C2[0] * x * S(4) + SH_C2[1] * z * S(5) + SH_C2[2] * 2.f * -y * S(6) + SH_C2[4] * 2.f * -y * S(8);
						dz3[ch] += SH_C2[1] * y * S(5) + SH_C2[2] * 2.f * 2.f * z * S(6) + SH_C2[3] * x * S(7);
					}
					if (s->D > 2) {
						SET(9, SH_C3[0] * y * (3.f * xx - yy)); SET(10, SH_C3[1] * xy * z); SET(11, SH_C3[2] * y * (4.f * zz - xx - yy));
						SET(12, SH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy)); SET(13, SH_C3[4] * x * (4.f * zz - xx - yy));
						SET(14, SH_C3[5] * z * (xx - yy)); SET(15, SH_C3[6] * x * (xx - 3.f * yy));
						for (int ch = 0; ch < 3; ch++) {
							dx3[ch] += (SH_C3[0] * S(9) * 3.f * 2.f * xy + SH_C3[1] * S(10) * yz + SH_C3[2] * S(11) * -2.f * xy + SH_C3[3] * S(12) * -3.f * 2.f * xz +
							            SH_C3[4] * S(13) * (-3.f * xx + 4.f * zz - yy) + SH_C3[5] * S(14) * 2.f * xz + SH_C3[6] * S(15) * 3.f * (xx - yy));
							dy3[ch] += (SH_C3[0] * S(9) * 3.f * (xx - yy) + SH_C3[1] * S(10) * xz + SH_C3[2] * S(11) * (-3.f * yy + 4.f * zz - xx) +
							            SH_C3[3] * S(12) * -3.f * 2.f * yz + SH_C3[4] * S(13) * -2.f * xy + SH_C3[5] * S(14) * -2.f * yz + SH_C3[6] * S(15) * -3.f * 2.f * xy);
							dz3[ch] += (SH_C3[1] * S(10) * xy + SH_C3[2] * S(11) * 4.f * 2.f * yz + SH_C3[3] * S(12) * 3.f * (2.f * zz - xx - yy) +
							            SH_C3[4] * S(13) * 4.f * 2.f * xz + SH_C3[5] * S(14) * (xx - yy));
						}
					}
				}
			}
#undef SET
#undef S
			const float ddir[3] = {dx3[0] * dRGB[0] + dx3[1] * dRGB[1] + dx3[2] * dRGB[2], dy3[0] * dRGB[0] + dy3[1] * dRGB[1] + dy3[2] * dRGB[2],
			                       dz3[0] * dRGB[0] + dz3[1] * dRGB[1] + dz3[2] * dRGB[2]};
			/* auxiliary.h:123-133 */
			const float sum2 = dor[0] * dor[0] + dor[1] * dor[1] + dor[2] * dor[2];
			const float inv32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
			dmean[0] += ((+sum2 - dor[0] * dor[0]) * ddir[0] - dor[1] * dor[0] * ddir[1] - dor[2] * dor[0] * ddir[2]) * inv32;
			dmean[1] += (-dor[0] * dor[1] * ddir[0] + (sum2 - dor[1] * dor[1]) * ddir[1] - dor[2] * dor[1] * ddir[2]) * inv32;
			dmean[2] += (-dor[0] * dor[2] * ddir[0] - dor[1] * dor[2] * ddir[1] + (sum2 - dor[2] * dor[2]) * ddir[2]) * inv32;
		}
		for (int i = 0; i < 3; i++) o->means3D[3 * idx + i] = dmean[i];
		/* backward.cu:492-555 */
		if (s->scales) {
			const float* q = s->rotations + 4 * idx; const float* scl = s->scales + 3 * idx;
			const float r = q[0], x = q[1], y = q[2], z = q[3];
			m3 R = m3_make(1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y), 2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z),
			               2.f * (y * z - r * x), 2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y));
			const float sv[3] = {s->scale_modifier * scl[0], s->scale_modifier * scl[1], s->scale_modifier * scl[2]};
			m3 S = m3_make(sv[0], 0, 0, 0, sv[1], 0, 0, 0, sv[2]);
			m3 Mm = m3_mul(S, R);
			m3 dSig = m3_make(dcov[0], 0.5f * dcov[1], 0.5f * dcov[2], 0.5f * dcov[1], dcov[3], 0.5f * dcov[4], 0.5f * dcov[2], 0.5f * dcov[4], dcov[5]);
			m3 dM = m3_mul(m3_scale(Mm, 2.0f), dSig);
			m3 Rt = m3_t(R), dMt = m3_t(dM);
			for (int k = 0; k < 3; k++) {
				v3 a3 = v3_make(Rt.c[k][0], Rt.c[k][1], Rt.c[k][2]), b3 = v3_make(dMt.c[k][0], dMt.c[k][1], dMt.c[k][2]);
				o->scales[3 * idx + k] = v3_dot(a3, b3);
				for (int rr = 0; rr < 3; rr++) dMt.c[k][rr] *= sv[k];
			}
#define Dm(cc, rr) dMt.c[cc][rr]
			float* dq = o->rotations + 4 * idx;
			dq[0] = 2 * z * (Dm(0, 1) - Dm(1, 0)) + 2 * y * (Dm(2, 0) - Dm(0, 2)) + 2 * x * (Dm(1, 2) - Dm(2, 1));
			dq[1] = 2 * y * (Dm(1, 0) + Dm(0, 1)) + 2 * z * (Dm(2, 0) + Dm(0, 2)) + 2 * r * (Dm(1, 2) - Dm(2, 1)) - 4 * x * (Dm(2, 2) + Dm(1, 1));
			dq[2] = 2 * x * (Dm(1, 0) + Dm(0, 1)) + 2 * r * (Dm(2, 0) - Dm(0, 2)) + 2 * z * (Dm(1, 2) + Dm(2, 1)) - 4 * y * (Dm(2, 2) + Dm(0, 0));
			dq[3] = 2 * r * (Dm(0, 1) - Dm(1, 0)) + 2 * x * (Dm(2, 0) + Dm(0, 2)) + 2 * y * (Dm(1, 2) + Dm(2, 1)) - 4 * z * (Dm(1, 1) + Dm(0, 0));
#undef Dm
		}
	}
}

/* ---- integrate_gaussians_to_points (SURVEY.md 8f row 3) ---------------------------------------------------------
 * computeCov2D<INTE> extras, forward.cu:187-235: the inverse covariance in (pixel x, pixel y, ray depth) space.  The
 * reference leaves it unassigned for ill-conditioned covariances (its else-branch fills a shadowed local, :214); those
 * Gaussians get condition = 0 and zeros here.  invraycov [P,6] must arrive zero-filled (rasterize_points.cu:317).
 * sigma_inv, if not NULL ([P,12], zero-filled), receives the Sigma^-1 each Gaussian in front of the near plane was given, in
 * the layout this build keeps it: 9 floats column-major, then the flag bits (1 well-conditioned, 2 solver converged). */
void orc_inte_geometry(const orc_scene* s, const orc_geom* g, float* invraycov, uint8_t* condition, float* sigma_inv) {
	const float focal_y = s->H / (2.0f * s->tan_fovy), focal_x = s->W / (2.0f * s->tan_fovx);
	const float* V = s->viewmatrix;
	for (int idx = 0; idx < s->P; idx++) {
		float pv[3]; xf4x3(s->means3D + 3 * idx, V, pv);
		if (pv[2] <= 0.2f) continue;
		const float* cov6 = g->cov3D + 6 * idx;
		float t[3] = {pv[0], pv[1], pv[2]};
		const float limx = 1.3f * s->tan_fovx, limy = 1.3f * s->tan_fovy;
		float txtz = t[0] / t[2], tytz = t[1] / t[2];
		t[0] = fminf2(limx, fmaxf2(-limx, txtz)) * t[2];
		t[1] = fminf2(limy, fmaxf2(-limy, tytz)) * t[2];
		txtz = t[0] / t[2]; tytz = t[1] / t[2];
		m3 Wm = m3_make(V[0], V[4], V[8], V[1], V[5], V[9], V[2], V[6], V[10]);
		sig_inv si = sigma_inverse(cov6);
		condition[idx] = (uint8_t)si.well;
		if (sigma_inv) {
			float* so = sigma_inv + 12 * idx;
			for (int c = 0; c < 3; c++) for (int k = 0; k < 3; k++) so[3 * c + k] = si.inv.c[c][k];
			const int32_t flags = (si.well ? 1 : 0) | (si.solved ? 2 : 0);
			memcpy(so + 9, &flags, sizeof(flags));
		}
		m3 cci = m3_mul(m3_mul(m3_t(Wm), si.inv), Wm);
		v3 uvh = v3_make(txtz, tytz, 1), uvh_mn = v3_normalize(m3_mulv(cci, uvh));
		if (isnan(uvh_mn.v[0]) || !si.solved || !si.well) continue;
		const float u2 = txtz * txtz, v2 = tytz * tytz, uv = txtz * tytz;
		const float l = sqrtf(t[0] * t[0] + t[1] * t[1] + t[2] * t[2]);
		const float ltz = u2 + v2 + 1;
		m3 full = m3_scale(m3_make(v2 + 1, -uv, txtz / l * ltz, -uv, u2 + 1, tytz / l * ltz, -txtz, -tytz, 1 / l * ltz), t[2] / (u2 + v2 + 1));
		m3 T2 = m3_mul(Wm, m3_t(full));
		m3 inv = m3_mul(m3_mul(m3_t(T2), si.inv), T2);
		m3 sc = m3_make(1 / focal_x, 0, 0, 0, 1 / focal_y, 0, 0, 0, 1);
		inv = m3_mul(m3_mul(sc, inv), sc);
		float* o = invraycov + 6 * idx;
		o[0] = inv.c[0][0]; o[1] = inv.c[0][1]; o[2] = inv.c[0][2]; o[3] = inv.c[1][1]; o[4] = inv.c[1][2]; o[5] = inv.c[2][2];
	}
}

#define ORC_MAX_CONTRIB (512 * 4)   /* MAX_NUM_CONTRIBUTORS * 4, auxiliary.h:31, forward.cu:1126 */

typedef struct {
	float* out_color;          /* [9,H,W], zero-filled by the caller */
	float* alpha_integrated;   /* [PN]  filled with 1      (rasterize_points.cu:313) */
	float* color_integrated;   /* [PN,3] filled with 0 */
	float* coordinate2d;       /* [PN,2] filled with 0 */
	float* sdf;                /* [PN]  filled with -1000 */
} orc_integrate_out;

/* forward.cu:938-1372 per pixel, serially.  Phase 1 renders with five sample positions (centre + corners) and records which
 * list entries contributed at any of them; phase 2 re-walks exactly those entries for every query point that projects
 * into the pixel, with the 3D (ray-space) Gaussian instead of the 2D conic.  Returns the number of pixels that hit the
 * contributor cap (the reference prints an error and stops that pixel). */
int orc_integrate(int W, int H, float tan_fovx, float tan_fovy, const float* bg, const uint32_t* ranges, const uint32_t* point_list,
                  const orc_geom* g, const float* invraycov, const uint8_t* condition, int PN, const float* points3D, const float* viewmatrix,
                  orc_integrate_out* o) {
	const int gx = (W + TILE - 1) / TILE;
	const float focal_y = H / (2.0f * tan_fovy), focal_x = W / (2.0f * tan_fovx);
	const size_t HW = (size_t)H * W;
	/* preprocessPointsCUDA (forward.cu:857-900): bucket the points by the pixel they fall into */
	float* pxy = (float*)malloc((size_t)PN * 2 * sizeof(float));
	float* pdepth = (float*)malloc((size_t)PN * sizeof(float));
	int* ppix = (int*)malloc((size_t)PN * sizeof(int));
	int* head = (int*)malloc((HW + 1) * sizeof(int));
	int* order = (int*)malloc((size_t)(PN > 0 ? PN : 1) * sizeof(int));
	memset(head, 0, (HW + 1) * sizeof(int));
	for (int i = 0; i < PN; i++) {
		ppix[i] = -1;
		float pv[3]; xf4x3(points3D + 3 * i, viewmatrix, pv);
		if (pv[2] <= 0.2f) continue;
		const float ix = (float)((double)(focal_x * pv[0] / (pv[2] + 0.0000001f)) + W / 2.);
		const float iy = (float)((double)(focal_y * pv[1] / (pv[2] + 0.0000001f)) + H / 2.);
		if (ix < 0 || ix >= W || iy < 0 || iy >= H) continue;
		pdepth[i] = sqrtf(pv[0] * pv[0] + pv[1] * pv[1] + pv[2] * pv[2]);
		pxy[2 * i] = ix; pxy[2 * i + 1] = iy;
		/* the pixel whose half-open box [x, x+1) x [y, y+1) holds the point (forward.cu:1212-1213) */
		ppix[i] = (int)iy * W + (int)ix;
		head[ppix[i] + 1]++;
	}
	for (size_t p = 0; p < HW; p++) head[p + 1] += head[p];
	{
		int* fill = (int*)malloc((HW + 1) * sizeof(int));
		memcpy(fill, head, (HW + 1) * sizeof(int));
		for (int i = 0; i < PN; i++) if (ppix[i] >= 0) order[fill[ppix[i]]++] = i;
		free(fill);
	}
	static const float off_x[5] = {0.0f, -0.5f, 0.5f, -0.5f, 0.5f}, off_y[5] = {0.0f, -0.5f, -0.5f, 0.5f, 0.5f};
	uint32_t* contributed = (uint32_t*)malloc(ORC_MAX_CONTRIB * sizeof(uint32_t));
	int overflowed = 0;
	for (int py = 0; py < H; py++) for (int px = 0; px < W; px++) {
		const size_t pix = (size_t)W * py + px;
		const float pxf = (float)px + 0.5f, pyf = (float)py + 0.5f;
		const uint32_t* rg = ranges + 2 * ((py / TILE) * gx + px / TILE);
		float T = 1.0f, C[8] = {0, 0, 0, 0, 0, 0, 0, 0};
		float mid_depth_center = 0, mid_plane[2] = {0, 0}, mid_mean2d[2] = {0, 0};
		float corner_T[5] = {1, 1, 1, 1, 1};
		uint32_t contributor = 0, last = 0; int n_contrib = 0;
		for (uint32_t it = rg[0]; it < rg[1]; it++) {
			contributor++;
			const int id = (int)point_list[it];
			const float* co = g->conic_opacity + 4 * id;
			const float depth_center = g->ts[id];
			const float plx = g->ray_planes[2 * id], ply = g->ray_planes[2 * id + 1];
			const float mx = g->means2D[2 * id], my = g->means2D[2 * id + 1];
			int used = 0;
			for (int k = 0; k < 5; k++) {
				const float dx = mx - pxf - off_x[k], dy = my - pyf - off_y[k];
				const float depth = depth_center + (plx * dx + ply * dy);
				const float power = -0.5f * (co[0] * dx * dx + co[2] * dy * dy) - co[1] * dx * dy;
				if (power > 0.0f) continue;
				const float alpha = fminf2(0.99f, co[3] * expf(power));
				if (alpha < 1.0f / 255.0f) continue;
				const float test_T = corner_T[k] * (1 - alpha);
				if (test_T < 0.0001f) continue;
				if (k == 0) for (int ch = 0; ch < 3; ch++) C[ch] += g->rgb[3 * id + ch] * alpha * T;
				if (depth > C[6]) C[6] = depth;
				if (k == 0) {
					C[7] += alpha * T;
					C[3] += depth * alpha * T;
					if (T > 0.5) { C[4] = depth; mid_depth_center = depth_center; mid_plane[0] = plx; mid_plane[1] = ply; mid_mean2d[0] = mx; mid_mean2d[1] = my; }
					T = test_T;
				}
				corner_T[k] = test_T;
				used = 1;
			}
			if (used) {
				last = contributor;
				contributed[n_contrib++] = contributor;
				if (n_contrib >= ORC_MAX_CONTRIB) { overflowed++; break; }
			}
		}
		for (int ch = 0; ch < 3; ch++) o->out_color[ch * HW + pix] = C[ch] + T * bg[ch];
		o->out_color[3 * HW + pix] = C[3];
		o->out_color[4 * HW + pix] = C[4];
		o->out_color[6 * HW + pix] = C[6];
		o->out_color[7 * HW + pix] = C[7];
		o->out_color[8 * HW + pix] = (float)(head[pix + 1] - head[pix]);
		(void)last;
		for (int q = head[pix]; q < head[pix + 1]; q++) {
			const int pid = order[q];
			const float qx = pxy[2 * pid], qy = pxy[2 * pid + 1], qdepth = pdepth[pid];
			float pa = 0.f, pT = 1.f;
			for (int c = 0; c < n_contrib; c++) {
				const int id = (int)point_list[rg[0] + contributed[c] - 1];
				const float* co = g->conic_opacity + 4 * id;
				const float depth_center = g->ts[id];
				const float dx = g->means2D[2 * id] - qx, dy = g->means2D[2 * id + 1] - qy;
				const float depth = depth_center + (g->ray_planes[2 * id] * dx + g->ray_planes[2 * id + 1] * dy);
				const float* ic = invraycov + 6 * id;
				float alpha;
				float dz;
				if (condition[id]) dz = depth_center - fminf2(qdepth, depth);
				else if (qdepth < depth) { continue; /* alpha = 0 */ }
				else dz = depth_center;
				{
					/* glm::dot(delta, M * delta), M symmetric from the six stored entries (forward.cu:1300-1312) */
					const float m0 = ic[0] * dx + ic[1] * dy + ic[2] * dz;
					const float m1 = ic[1] * dx + ic[3] * dy + ic[4] * dz;
					const float m2 = ic[2] * dx + ic[4] * dy + ic[5] * dz;
					const float power = -0.5f * (dx * m0 + dy * m1 + dz * m2);
					alpha = fminf2(0.99f, co[3] * expf(power));
				}
				if (alpha < 1.0f / 255.0f) continue;
				pa += alpha * pT;
				pT = pT * (1 - alpha);
			}
			o->alpha_integrated[pid] = pa;
			for (int ch = 0; ch < 3; ch++) o->color_integrated[3 * pid + ch] = C[ch] + T * bg[ch];
			o->coordinate2d[2 * pid] = qx; o->coordinate2d[2 * pid + 1] = qy;
			if (qdepth > 0) {
				const float dx = mid_mean2d[0] - qx, dy = mid_mean2d[1] - qy;
				o->sdf[pid] = (mid_depth_center + (mid_plane[0] * dx + mid_plane[1] * dy)) - qdepth;
			}
		}
	}
	free(contributed); free(order); free(head); free(ppix); free(pdepth); free(pxy);
	return overflowed;
}
