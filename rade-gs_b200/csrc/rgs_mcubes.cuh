// rgs_mcubes.cuh -- the marching-cubes triangle table shared by the sparse TSDF mesh (rgs_tsdf.cu) and the dense crops of
// the unbounded mesh (rgs_unbounded.cu).  The table is derived at compile time from the watertight face rule stated at
// rgs_tsdf_* in include/rgs_b200.h: corner c = x + 2y + 4z, case bit c set when corner c is inside, edge e runs along axis
// e / 4 from the corner offset by (e & 1, e >> 1 & 1) on the other two axes; the right-hand normal of every triangle points
// toward increasing field values.
#pragma once
#include <stdint.h>

namespace rgs {

struct TriTable {
	int8_t n[256];          // triangles per case
	int8_t e[256][15];      // edges, 3 per triangle
	bool ok;                // every sign-change edge has one segment out and one in (closed loops)
};

constexpr int other_axis(int a, int k) { return k == 0 ? (a == 0 ? 1 : 0) : (a == 2 ? 1 : 2); }
// corner of edge e at its end `hi` (0 / 1 along the edge's axis), as x + 2y + 4z
constexpr int edge_corner(int e, int hi) {
	const int a = e / 4, o = e % 4;
	int p[3] = {0, 0, 0};
	p[other_axis(a, 0)] = o & 1;
	p[other_axis(a, 1)] = o >> 1 & 1;
	p[a] = hi;
	return p[0] + 2 * p[1] + 4 * p[2];
}
constexpr int corner_coord(int c, int k) { return c >> k & 1; }

constexpr TriTable make_tri_table() {
	TriTable t{};
	t.ok = true;
	for (int cs = 0; cs < 256; cs++) {
		int succ[12] = {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1};
		int pred[12] = {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1};
		bool change[12] = {};
		for (int e = 0; e < 12; e++) change[e] = ((cs >> edge_corner(e, 0)) & 1) != ((cs >> edge_corner(e, 1)) & 1);
		for (int a = 0; a < 3; a++) {
			for (int s = 0; s < 2; s++) {
				int fe[4] = {}, nf = 0, ch[4] = {}, nc = 0;
				for (int e = 0; e < 12; e++)
					if (e / 4 != a && corner_coord(edge_corner(e, 0), a) == s) {
						fe[nf++] = e;
						if (change[e]) ch[nc++] = e;
					}
				int segs[2][2] = {}, ns = 0;
				if (nc == 2) {
					segs[0][0] = ch[0];
					segs[0][1] = ch[1];
					ns = 1;
				} else if (nc == 4) {  // ambiguous face: each inside corner is cut off by the segment of its two face edges
					for (int c = 0; c < 8; c++) {
						if (corner_coord(c, a) != s || !((cs >> c) & 1)) continue;
						int k = 0;
						for (int i = 0; i < 4; i++)
							if (edge_corner(fe[i], 0) == c || edge_corner(fe[i], 1) == c) segs[ns][k++] = fe[i];
						ns++;
					}
				} else if (nc != 0) {
					t.ok = false;
				}
				for (int q = 0; q < ns; q++) {
					int A = segs[q][0], B = segs[q][1];
					// doubled midpoints, inside corner of A (doubled), outward normal of the face
					int ma[3] = {}, mb[3] = {}, in[3] = {}, n[3] = {};
					const int ia = ((cs >> edge_corner(A, 0)) & 1) ? edge_corner(A, 0) : edge_corner(A, 1);
					for (int k = 0; k < 3; k++) {
						ma[k] = corner_coord(edge_corner(A, 0), k) + corner_coord(edge_corner(A, 1), k);
						mb[k] = corner_coord(edge_corner(B, 0), k) + corner_coord(edge_corner(B, 1), k);
						in[k] = 2 * corner_coord(ia, k) - ma[k];
					}
					n[a] = s ? 1 : -1;
					const int d[3] = {mb[0] - ma[0], mb[1] - ma[1], mb[2] - ma[2]};
					const int x[3] = {d[1] * n[2] - d[2] * n[1], d[2] * n[0] - d[0] * n[2], d[0] * n[1] - d[1] * n[0]};
					if (x[0] * in[0] + x[1] * in[1] + x[2] * in[2] < 0) {
						const int tmp = A;
						A = B;
						B = tmp;
					}
					if (succ[A] != -1 || pred[B] != -1) t.ok = false;
					succ[A] = B;
					pred[B] = A;
				}
			}
		}
		bool seen[12] = {};
		int nt = 0;
		for (int e = 0; e < 12; e++) {
			if (!change[e] || seen[e]) continue;
			if (succ[e] < 0 || pred[e] < 0) { t.ok = false; break; }
			int loop[12] = {}, len = 0, cur = e;
			do {
				if (len == 12 || cur < 0) { t.ok = false; break; }
				loop[len++] = cur;
				seen[cur] = true;
				cur = succ[cur];
			} while (cur != e);
			for (int k = 1; k + 1 < len; k++) {
				if (nt == 5) { t.ok = false; break; }
				t.e[cs][3 * nt] = (int8_t)loop[0];
				t.e[cs][3 * nt + 1] = (int8_t)loop[k];
				t.e[cs][3 * nt + 2] = (int8_t)loop[k + 1];
				nt++;
			}
		}
		t.n[cs] = (int8_t)nt;
	}
	return t;
}

constexpr TriTable kTriTable = make_tri_table();
static_assert(kTriTable.ok, "triangle table: the face segments do not close into loops");
static_assert(kTriTable.n[0] == 0 && kTriTable.n[255] == 0 && kTriTable.n[1] == 1, "triangle table: trivial cases");
// one copy per translation unit that includes this header
static __constant__ TriTable c_tri = kTriTable;

}  // namespace rgs
