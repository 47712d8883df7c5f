/* render_oracle.c -- fp64 CPU ray caster for the depth renderer (clean_pvnet_b200/csrc/render.cu, DESIGN.md 8f).
 *
 * TEST INFRASTRUCTURE ONLY.  It is written from the renderer's stated semantics, not from any OpenGL code: pixel
 * (row r, column c) casts the camera ray through (u, v) = (c + 0.5, r + 0.5) of the intrinsics
 * u = fx X/Z + s Y/Z + cx, v = fy Y/Z + cy, intersects it with every triangle (Moller-Trumbore, in the camera frame) and
 * keeps the nearest hit whose Z lies in [near, far].  The device kernel uses a different formulation (homogeneous edge
 * functions in K-space), so agreement is evidence for both.
 *
 * Per pixel it returns:
 *   z     the nearest hit Z in [near, far], or 0
 *   edge  the screen-space distance from the pixel centre to the boundary of any projected triangle whose plane the ray
 *         meets within [near, far] no farther than z (every such triangle when nothing is hit), i.e. to the nearest edge
 *         line of a triangle it is inside and the nearest edge segment of one it is outside (the edge line when a vertex
 *         is behind the camera): the pixels where a rounding of the coverage test could change the answer
 *   gap   second-nearest hit Z minus z (inf when fewer than two hits): where a rounding could change the winner
 *   clip  the smallest |Z - near| or |Z - far| over the triangles the ray passes through (inf if none): where a rounding
 *         could change the clip test
 * Model points and the pose are taken as given (the caller rounds them to fp32 as the device does).
 */
#include <math.h>
#include <stdlib.h>

#define API __attribute__((visibility("default")))

typedef struct { double x, y, z; } v3;

static v3 sub(v3 a, v3 b) { v3 r = {a.x - b.x, a.y - b.y, a.z - b.z}; return r; }
static v3 cross(v3 a, v3 b) { v3 r = {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; return r; }
static double dot(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

/* ray parameter t (= Z, the ray's z component is 1) and barycentrics of the ray's meeting with the triangle's plane;
 * returns 0 for a plane parallel to the ray */
static int intersect(v3 d, v3 p0, v3 p1, v3 p2, double *t, double *b1, double *b2)
{
    v3 e1 = sub(p1, p0), e2 = sub(p2, p0), pv = cross(d, e2);
    double det = dot(e1, pv);
    if (det == 0.0 || !isfinite(det)) return 0;
    double inv = 1.0 / det;
    v3 tv = {-p0.x, -p0.y, -p0.z};
    v3 qv = cross(tv, e1);
    *b1 = dot(tv, pv) * inv;
    *b2 = dot(d, qv) * inv;
    *t = dot(e2, qv) * inv;
    return 1;
}

API void orc_render_depth(const float *pts, int V, const int *faces, int F, const double *pose, const double *K, int H,
                          int W, double znear, double zfar, double *z_out, double *edge_out, double *gap_out,
                          double *clip_out)
{
    double fx = K[0], s = K[1], cx = K[2], fy = K[4], cy = K[5];
    v3 *P = malloc(sizeof(v3) * (V > 0 ? V : 1));
    int *box = malloc(sizeof(int) * 4 * (F > 0 ? F : 1));
    for (int i = 0; i < V; ++i) {
        double x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
        P[i].x = pose[0] * x + pose[1] * y + pose[2] * z + pose[3];
        P[i].y = pose[4] * x + pose[5] * y + pose[6] * z + pose[7];
        P[i].z = pose[8] * x + pose[9] * y + pose[10] * z + pose[11];
    }
    /* conservative pixel boxes: the projected vertices' box plus one pixel, the whole image when a vertex is not in
     * front of the near plane */
    for (int f = 0; f < F; ++f) {
        int *b = box + 4 * f;
        double u0 = INFINITY, u1 = -INFINITY, v0 = INFINITY, v1 = -INFINITY;
        int whole = 0;
        for (int j = 0; j < 3; ++j) {
            v3 q = P[faces[3 * f + j]];
            if (!(q.z >= znear)) { whole = 1; break; }
            double u = (fx * q.x + s * q.y) / q.z + cx, v = fy * q.y / q.z + cy;
            u0 = fmin(u0, u); u1 = fmax(u1, u); v0 = fmin(v0, v); v1 = fmax(v1, v);
        }
        if (whole) { b[0] = 0; b[1] = W - 1; b[2] = 0; b[3] = H - 1; continue; }
        b[0] = (int)fmax(0.0, floor(u0) - 1); b[1] = (int)fmin(W - 1.0, ceil(u1) + 1);
        b[2] = (int)fmax(0.0, floor(v0) - 1); b[3] = (int)fmin(H - 1.0, ceil(v1) + 1);
    }
    for (int i = 0; i < H * W; ++i) { z_out[i] = INFINITY; gap_out[i] = INFINITY; edge_out[i] = INFINITY; clip_out[i] = INFINITY; }
    double *second = malloc(sizeof(double) * (H * W > 0 ? H * W : 1));
    for (int i = 0; i < H * W; ++i) second[i] = INFINITY;
    /* pass 1: nearest and second-nearest hits, clip margins */
    for (int f = 0; f < F; ++f) {
        const int *b = box + 4 * f;
        v3 p0 = P[faces[3 * f]], p1 = P[faces[3 * f + 1]], p2 = P[faces[3 * f + 2]];
        for (int r = b[2]; r <= b[3]; ++r)
            for (int c = b[0]; c <= b[1]; ++c) {
                double u = c + 0.5, v = r + 0.5, t, b1, b2;
                double yv = (v - cy) / fy;
                v3 d = {(u - cx - s * yv) / fx, yv, 1.0};
                if (!intersect(d, p0, p1, p2, &t, &b1, &b2)) continue;
                if (!(b1 >= 0.0 && b2 >= 0.0 && b1 + b2 <= 1.0 && t > 0.0)) continue;
                int i = r * W + c;
                double m = fmin(fabs(t - znear), fabs(t - zfar));
                if (m < clip_out[i]) clip_out[i] = m;
                if (!(t >= znear && t <= zfar)) continue;
                if (t < z_out[i]) { second[i] = z_out[i]; z_out[i] = t; }
                else if (t < second[i]) second[i] = t;
            }
    }
    /* pass 2: edge margins of every triangle that could take the pixel */
    for (int f = 0; f < F; ++f) {
        const int *b = box + 4 * f;
        v3 q[3];
        for (int j = 0; j < 3; ++j) {
            v3 p = P[faces[3 * f + j]];
            q[j].x = fx * p.x + s * p.y + cx * p.z; q[j].y = fy * p.y + cy * p.z; q[j].z = p.z;
        }
        v3 l[3] = {cross(q[0], q[1]), cross(q[1], q[2]), cross(q[2], q[0])};
        v3 p0 = P[faces[3 * f]], p1 = P[faces[3 * f + 1]], p2 = P[faces[3 * f + 2]];
        int front = p0.z > 0.0 && p1.z > 0.0 && p2.z > 0.0;
        for (int r = b[2]; r <= b[3]; ++r)
            for (int c = b[0]; c <= b[1]; ++c) {
                double u = c + 0.5, v = r + 0.5, t, b1, b2;
                double yv = (v - cy) / fy;
                v3 d = {(u - cx - s * yv) / fx, yv, 1.0};
                if (!intersect(d, p0, p1, p2, &t, &b1, &b2)) continue;
                int i = r * W + c;
                if (!(t >= znear && t <= zfar) || t > z_out[i]) continue;
                v3 x = {u, v, 1.0};
                int inside = b1 >= 0.0 && b2 >= 0.0 && b1 + b2 <= 1.0;
                for (int j = 0; j < 3; ++j) {
                    /* inside: the distance to the boundary is the nearest edge line's; outside and in front of the
                     * camera: the distance to the projected triangle, i.e. to the nearest edge segment */
                    double m = fabs(dot(l[j], x)) / hypot(l[j].x, l[j].y);
                    if (!inside && front) {
                        v3 a = q[j], b = q[(j + 1) % 3];
                        double ax = a.x / a.z, ay = a.y / a.z, bx = b.x / b.z, by = b.y / b.z;
                        double ex = bx - ax, ey = by - ay, len2 = ex * ex + ey * ey;
                        double s = len2 > 0.0 ? ((u - ax) * ex + (v - ay) * ey) / len2 : 0.0;
                        s = s < 0.0 ? 0.0 : s > 1.0 ? 1.0 : s;
                        m = hypot(u - (ax + s * ex), v - (ay + s * ey));
                    }
                    if (m < edge_out[i]) edge_out[i] = m;
                }
            }
    }
    for (int i = 0; i < H * W; ++i) {
        gap_out[i] = isfinite(z_out[i]) ? second[i] - z_out[i] : INFINITY;
        if (!isfinite(z_out[i])) z_out[i] = 0.0;
    }
    free(second); free(box); free(P);
}
