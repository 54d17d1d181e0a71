// host_scene.cpp -- the CPU scene pipeline that feeds the hot path (north_star: "C++ host
// code loads the OBJ meshes and builds the SAH BVH on CPU exactly as the reference does").
//
// Restates, behind the C ABI of include/ezrt.h:
//   getTransformMatrix   P5/main.cpp:255-271      readObj           P5/main.cpp:274-392
//   buildBVH             P5/main.cpp:395-455      buildBVHwithSAH   P5/main.cpp:458-589
//   scene encode         P5/main.cpp:843-871      HDRLoader::load   P5/lib/hdrloader.cpp:29-97
//   calculateHdrCache    P5/main.cpp:592-689      display() camera  P5/main.cpp:710-713
// glm (not vendored by the reference, no version pin) is restated on top of ezrt_math.h;
// the operation orders of mat4*vec4, mat4*mat4, rotate, lookAt and inverse follow glm 0.9.9.
//
// Compile with -ffp-contract=off -mfma (see __graft_entry__.build()).
#include "ezrt.h"
#include "ezrt_math.h"
#include "ezrt_internal.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <future>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

namespace {

// ------------------------------------------------------------------------------------------
// data (P5/main.cpp:27-56)
// ------------------------------------------------------------------------------------------
struct Tri {
    ez_vec3 p1, p2, p3;
    ez_vec3 n1, n2, n3;
    float material[EZRT_MATERIAL_FLOATS];
    // base-colour texture (ezrt_trilist_read_obj_textured): (u1, v1, u2, v2, u3, v3) and the texture id, -1 = untextured.  Carried
    // through every builder: the builders' permutations depend only on comparison outcomes, never on these
    float uv[6] = {0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f};
    int32_t tex_id = -1;
};
struct Node {
    int left, right, n, index;
    ez_vec3 AA, BB;
};

struct Mat4 {
    float c[4][4];  // c[col][row], glm layout
};

Mat4 mat_identity() {
    Mat4 m;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) m.c[i][j] = (i == j) ? 1.0f : 0.0f;
    return m;
}

// glm operator*(mat4, mat4): Result[i] = A0*B[i][0] + A1*B[i][1] + A2*B[i][2] + A3*B[i][3]
Mat4 mat_mul(const Mat4& a, const Mat4& b) {
    Mat4 r;
    for (int i = 0; i < 4; i++)
        for (int k = 0; k < 4; k++)
            r.c[i][k] = ((a.c[0][k] * b.c[i][0] + a.c[1][k] * b.c[i][1]) + a.c[2][k] * b.c[i][2]) +
                        a.c[3][k] * b.c[i][3];
    return r;
}

// glm operator*(mat4, vec4): (m0*v.x + m1*v.y) + (m2*v.z + m3*v.w)
void mat_mul_vec4(const Mat4& m, const float v[4], float out[4]) {
    for (int k = 0; k < 4; k++) {
        float a0 = m.c[0][k] * v[0] + m.c[1][k] * v[1];
        float a1 = m.c[2][k] * v[2] + m.c[3][k] * v[3];
        out[k] = a0 + a1;
    }
}

const float kDegToRad = 0.01745329251994329576923690768489f;  // glm::radians

// glm::rotate(m, angle, axis) for a unit axis
Mat4 mat_rotate(const Mat4& m, float angle, ez_vec3 v) {
    float c = ez_cos(angle);
    float s = ez_sin(angle);
    ez_vec3 axis = ez_normalize(v);
    ez_vec3 temp = ez_scale(axis, 1.0f - c);
    float R[3][3];
    R[0][0] = c + temp.x * axis.x;
    R[0][1] = temp.x * axis.y + s * axis.z;
    R[0][2] = temp.x * axis.z - s * axis.y;
    R[1][0] = temp.y * axis.x - s * axis.z;
    R[1][1] = c + temp.y * axis.y;
    R[1][2] = temp.y * axis.z + s * axis.x;
    R[2][0] = temp.z * axis.x + s * axis.y;
    R[2][1] = temp.z * axis.y - s * axis.x;
    R[2][2] = c + temp.z * axis.z;
    Mat4 r;
    for (int i = 0; i < 3; i++)
        for (int k = 0; k < 4; k++)
            r.c[i][k] = (m.c[0][k] * R[i][0] + m.c[1][k] * R[i][1]) + m.c[2][k] * R[i][2];
    for (int k = 0; k < 4; k++) r.c[3][k] = m.c[3][k];
    return r;
}

// getTransformMatrix, P5/main.cpp:255-271
Mat4 transform_matrix(const float rot[3], const float tr[3], const float sc[3]) {
    Mat4 unit = mat_identity();
    Mat4 scale = unit;
    for (int k = 0; k < 4; k++) {
        scale.c[0][k] = unit.c[0][k] * sc[0];
        scale.c[1][k] = unit.c[1][k] * sc[1];
        scale.c[2][k] = unit.c[2][k] * sc[2];
    }
    Mat4 translate = unit;
    for (int k = 0; k < 4; k++)
        translate.c[3][k] = ((unit.c[0][k] * tr[0] + unit.c[1][k] * tr[1]) + unit.c[2][k] * tr[2]) + unit.c[3][k];
    Mat4 rotate = unit;
    rotate = mat_rotate(rotate, rot[0] * kDegToRad, ez_v3(1, 0, 0));
    rotate = mat_rotate(rotate, rot[1] * kDegToRad, ez_v3(0, 1, 0));
    rotate = mat_rotate(rotate, rot[2] * kDegToRad, ez_v3(0, 0, 1));
    return mat_mul(mat_mul(translate, rotate), scale);
}

// glm::inverse(mat4) (cofactor expansion, glm/detail/func_matrix.inl)
Mat4 mat_inverse(const Mat4& M) {
    const float(*m)[4] = M.c;
    float Coef00 = m[2][2] * m[3][3] - m[3][2] * m[2][3];
    float Coef02 = m[1][2] * m[3][3] - m[3][2] * m[1][3];
    float Coef03 = m[1][2] * m[2][3] - m[2][2] * m[1][3];
    float Coef04 = m[2][1] * m[3][3] - m[3][1] * m[2][3];
    float Coef06 = m[1][1] * m[3][3] - m[3][1] * m[1][3];
    float Coef07 = m[1][1] * m[2][3] - m[2][1] * m[1][3];
    float Coef08 = m[2][1] * m[3][2] - m[3][1] * m[2][2];
    float Coef10 = m[1][1] * m[3][2] - m[3][1] * m[1][2];
    float Coef11 = m[1][1] * m[2][2] - m[2][1] * m[1][2];
    float Coef12 = m[2][0] * m[3][3] - m[3][0] * m[2][3];
    float Coef14 = m[1][0] * m[3][3] - m[3][0] * m[1][3];
    float Coef15 = m[1][0] * m[2][3] - m[2][0] * m[1][3];
    float Coef16 = m[2][0] * m[3][2] - m[3][0] * m[2][2];
    float Coef18 = m[1][0] * m[3][2] - m[3][0] * m[1][2];
    float Coef19 = m[1][0] * m[2][2] - m[2][0] * m[1][2];
    float Coef20 = m[2][0] * m[3][1] - m[3][0] * m[2][1];
    float Coef22 = m[1][0] * m[3][1] - m[3][0] * m[1][1];
    float Coef23 = m[1][0] * m[2][1] - m[2][0] * m[1][1];
    float Fac0[4] = {Coef00, Coef00, Coef02, Coef03};
    float Fac1[4] = {Coef04, Coef04, Coef06, Coef07};
    float Fac2[4] = {Coef08, Coef08, Coef10, Coef11};
    float Fac3[4] = {Coef12, Coef12, Coef14, Coef15};
    float Fac4[4] = {Coef16, Coef16, Coef18, Coef19};
    float Fac5[4] = {Coef20, Coef20, Coef22, Coef23};
    float Vec0[4] = {m[1][0], m[0][0], m[0][0], m[0][0]};
    float Vec1[4] = {m[1][1], m[0][1], m[0][1], m[0][1]};
    float Vec2[4] = {m[1][2], m[0][2], m[0][2], m[0][2]};
    float Vec3[4] = {m[1][3], m[0][3], m[0][3], m[0][3]};
    const float SignA[4] = {+1, -1, +1, -1};
    const float SignB[4] = {-1, +1, -1, +1};
    Mat4 Inv;
    for (int k = 0; k < 4; k++) {
        float Inv0 = (Vec1[k] * Fac0[k] - Vec2[k] * Fac1[k]) + Vec3[k] * Fac2[k];
        float Inv1 = (Vec0[k] * Fac0[k] - Vec2[k] * Fac3[k]) + Vec3[k] * Fac4[k];
        float Inv2 = (Vec0[k] * Fac1[k] - Vec1[k] * Fac3[k]) + Vec3[k] * Fac5[k];
        float Inv3 = (Vec0[k] * Fac2[k] - Vec1[k] * Fac4[k]) + Vec2[k] * Fac5[k];
        Inv.c[0][k] = Inv0 * SignA[k];
        Inv.c[1][k] = Inv1 * SignB[k];
        Inv.c[2][k] = Inv2 * SignA[k];
        Inv.c[3][k] = Inv3 * SignB[k];
    }
    float Dot0[4];
    for (int k = 0; k < 4; k++) Dot0[k] = m[0][k] * Inv.c[k][0];
    float Dot1 = (Dot0[0] + Dot0[1]) + (Dot0[2] + Dot0[3]);
    float OneOverDeterminant = 1.0f / Dot1;
    for (int i = 0; i < 4; i++)
        for (int k = 0; k < 4; k++) Inv.c[i][k] = Inv.c[i][k] * OneOverDeterminant;
    return Inv;
}

// glm::lookAt (right-handed)
Mat4 mat_look_at(ez_vec3 eye, ez_vec3 center, ez_vec3 up) {
    ez_vec3 f = ez_normalize(ez_sub(center, eye));
    ez_vec3 s = ez_normalize(ez_cross(f, up));
    ez_vec3 u = ez_cross(s, f);
    Mat4 r = mat_identity();
    r.c[0][0] = s.x; r.c[1][0] = s.y; r.c[2][0] = s.z;
    r.c[0][1] = u.x; r.c[1][1] = u.y; r.c[2][1] = u.z;
    r.c[0][2] = -f.x; r.c[1][2] = -f.y; r.c[2][2] = -f.z;
    r.c[3][0] = -ez_dot(s, eye);
    r.c[3][1] = -ez_dot(u, eye);
    r.c[3][2] = ez_dot(f, eye);
    return r;
}

// ------------------------------------------------------------------------------------------
// readObj, P5/main.cpp:274-392
// ------------------------------------------------------------------------------------------
// textured (ezrt_trilist_read_obj_textured): also the "vt u v [w]" lines and each face vertex's vt index; a triangle whose three
// vertices all carry one gets (its UVs, texture_id), any other -1.  Positions, normals and materials are read_obj's.
int read_obj_stream(std::istream& fin, std::vector<Tri>& triangles, const float material[EZRT_MATERIAL_FLOATS],
                    const Mat4& trans, bool smoothNormal, bool hardened = false, bool textured = false, int texture_id = -1) {
    std::vector<ez_vec3> vertices;
    std::vector<unsigned> indices;
    std::vector<float> texcoords;   // textured: 2 floats per vt line
    std::vector<int> tri_vt;        // textured: 3 vt indices (0-based) per triangle, or -1 when a vertex has none

    float maxx = -11451419.19f, maxy = -11451419.19f, maxz = -11451419.19f;
    float minx = 11451419.19f, miny = 11451419.19f, minz = 11451419.19f;

    std::string line;
    while (std::getline(fin, line)) {
        std::istringstream sin(line);
        std::string type;
        sin >> type;
        if (type == "v") {
            float x = 0, y = 0, z = 0;
            sin >> x >> y >> z;
            vertices.push_back(ez_v3(x, y, z));
            // the reference's normalisation quirk: maxy/maxz/miny/minz are fed from maxx/minx (:317-318)
            maxx = ez_max(maxx, x); maxy = ez_max(maxx, y); maxz = ez_max(maxx, z);
            minx = ez_min(minx, x); miny = ez_min(minx, y); minz = ez_min(minx, z);
        }
        if (textured && type == "vt") {   // a third component is ignored
            float u = 0, v = 0;
            sin >> u >> v;
            texcoords.push_back(u);
            texcoords.push_back(v);
        }
        if (type == "f") {
            // "v", "v/vt", "v/vt/vn" (and, hardened, "v//vn"): the leading integer of each
            // of the first three vertex tokens; extra vertices are ignored as in the reference.
            // Hardened mode (EZRT_OBJ_HARDENED): negative (relative) indices, and polygons are
            // triangulated as a fan instead of being cut to their first three vertices.
            std::vector<int> fv, fvt;
            std::string tok;
            while (sin >> tok) {
                char* end = nullptr;
                int idx = (int)std::strtol(tok.c_str(), &end, 10);
                if (hardened && idx < 0) idx = (int)vertices.size() + 1 + idx;
                fv.push_back(idx);
                if (textured) {   // "v/vt[/vn]": the integer after the first '/', if any (0 = none)
                    int vt = 0;
                    if (*end == '/' && end[1] != '/' && end[1] != '\0') {
                        vt = (int)std::strtol(end + 1, nullptr, 10);
                        if (hardened && vt < 0) vt = (int)(texcoords.size() / 2) + 1 + vt;
                        if (vt < 1) return EZRT_ERR_IO;
                    }
                    fvt.push_back(vt);
                }
                if (!hardened && fv.size() == 3) break;
            }
            if (fv.size() < 3) return EZRT_ERR_IO;
            for (int idx : fv)
                if (idx < 1) return EZRT_ERR_IO;   // upper bound: after the whole file is read (a face may precede its vertices)
            const bool face_vt = textured && std::find(fvt.begin(), fvt.end(), 0) == fvt.end();
            for (size_t k = 2; k < fv.size(); k++) {
                indices.push_back((unsigned)(fv[0] - 1));
                indices.push_back((unsigned)(fv[k - 1] - 1));
                indices.push_back((unsigned)(fv[k] - 1));
                if (textured) {
                    tri_vt.push_back(face_vt ? fvt[0] - 1 : -1);
                    tri_vt.push_back(face_vt ? fvt[k - 1] - 1 : -1);
                    tri_vt.push_back(face_vt ? fvt[k] - 1 : -1);
                }
            }
        }
    }

    for (unsigned idx : indices)   // the reference resolves indices after reading the whole file (P5/main.cpp:344-362)
        if ((size_t)idx >= vertices.size()) return EZRT_ERR_IO;
    for (int vt : tri_vt)
        if (vt >= 0 && (size_t)vt >= texcoords.size() / 2) return EZRT_ERR_IO;

    float lenx = maxx - minx, leny = maxy - miny, lenz = maxz - minz;
    float maxaxis = ez_max(lenx, ez_max(leny, lenz));
    for (auto& v : vertices) {
        v.x /= maxaxis; v.y /= maxaxis; v.z /= maxaxis;
    }
    for (auto& v : vertices) {
        float vv[4] = {v.x, v.y, v.z, 1.0f}, o[4];
        mat_mul_vec4(trans, vv, o);
        v = ez_v3(o[0], o[1], o[2]);
    }

    std::vector<ez_vec3> normals(vertices.size(), ez_v3(0, 0, 0));
    for (size_t i = 0; i + 2 < indices.size(); i += 3) {
        ez_vec3 p1 = vertices[indices[i]], p2 = vertices[indices[i + 1]], p3 = vertices[indices[i + 2]];
        ez_vec3 n = ez_normalize(ez_cross(ez_sub(p2, p1), ez_sub(p3, p1)));
        normals[indices[i]] = ez_add(normals[indices[i]], n);
        normals[indices[i + 1]] = ez_add(normals[indices[i + 1]], n);
        normals[indices[i + 2]] = ez_add(normals[indices[i + 2]], n);
    }

    size_t offset = triangles.size();
    triangles.resize(offset + indices.size() / 3);
    for (size_t i = 0; i + 2 < indices.size(); i += 3) {
        Tri& t = triangles[offset + i / 3];
        t.p1 = vertices[indices[i]];
        t.p2 = vertices[indices[i + 1]];
        t.p3 = vertices[indices[i + 2]];
        if (!smoothNormal) {
            ez_vec3 n = ez_normalize(ez_cross(ez_sub(t.p2, t.p1), ez_sub(t.p3, t.p1)));
            t.n1 = n; t.n2 = n; t.n3 = n;
        } else {
            t.n1 = ez_normalize(normals[indices[i]]);
            t.n2 = ez_normalize(normals[indices[i + 1]]);
            t.n3 = ez_normalize(normals[indices[i + 2]]);
        }
        memcpy(t.material, material, sizeof(t.material));
        if (textured && tri_vt[i] >= 0) {
            for (int c = 0; c < 3; c++) {
                t.uv[2 * c] = texcoords[2 * (size_t)tri_vt[i + c]];
                t.uv[2 * c + 1] = texcoords[2 * (size_t)tri_vt[i + c] + 1];
            }
            t.tex_id = texture_id;
        }
    }
    return EZRT_OK;
}

// ------------------------------------------------------------------------------------------
// BVH builders
// ------------------------------------------------------------------------------------------
inline ez_vec3 centroid(const Tri& t) {  // cmpx/cmpy/cmpz, P5/main.cpp:156-170
    return ez_divs(ez_add(ez_add(t.p1, t.p2), t.p3), 3.0f);
}
bool cmpx(const Tri& a, const Tri& b) { return centroid(a).x < centroid(b).x; }
bool cmpy(const Tri& a, const Tri& b) { return centroid(a).y < centroid(b).y; }
bool cmpz(const Tri& a, const Tri& b) { return centroid(a).z < centroid(b).z; }

inline ez_vec3 tri_min(const Tri& t) {
    return ez_v3(ez_min(t.p1.x, ez_min(t.p2.x, t.p3.x)), ez_min(t.p1.y, ez_min(t.p2.y, t.p3.y)),
                 ez_min(t.p1.z, ez_min(t.p2.z, t.p3.z)));
}
inline ez_vec3 tri_max(const Tri& t) {
    return ez_v3(ez_max(t.p1.x, ez_max(t.p2.x, t.p3.x)), ez_max(t.p1.y, ez_max(t.p2.y, t.p3.y)),
                 ez_max(t.p1.z, ez_max(t.p2.z, t.p3.z)));
}

void node_init(Node& nd) {
    nd.left = nd.right = nd.n = nd.index = 0;
    nd.AA = ez_v3(1145141919.0f, 1145141919.0f, 1145141919.0f);
    nd.BB = ez_v3(-1145141919.0f, -1145141919.0f, -1145141919.0f);
}

// buildBVH, P5/main.cpp:395-455 (median split on the longest axis)
int build_median(std::vector<Tri>& tris, std::vector<Node>& nodes, int l, int r, int n) {
    if (l > r) return 0;
    nodes.push_back(Node());
    int id = (int)nodes.size() - 1;
    node_init(nodes[id]);
    for (int i = l; i <= r; i++) {
        nodes[id].AA = ez_vmin(nodes[id].AA, tri_min(tris[i]));
        nodes[id].BB = ez_vmax(nodes[id].BB, tri_max(tris[i]));
    }
    if ((r - l + 1) <= n) {
        nodes[id].n = r - l + 1;
        nodes[id].index = l;
        return id;
    }
    float lenx = nodes[id].BB.x - nodes[id].AA.x;
    float leny = nodes[id].BB.y - nodes[id].AA.y;
    float lenz = nodes[id].BB.z - nodes[id].AA.z;
    if (lenx >= leny && lenx >= lenz) std::sort(tris.begin() + l, tris.begin() + r + 1, cmpx);
    if (leny >= lenx && leny >= lenz) std::sort(tris.begin() + l, tris.begin() + r + 1, cmpy);
    if (lenz >= lenx && lenz >= leny) std::sort(tris.begin() + l, tris.begin() + r + 1, cmpz);
    int mid = (l + r) / 2;
    int left = build_median(tris, nodes, l, mid, n);
    int right = build_median(tris, nodes, mid + 1, r, n);
    nodes[id].left = left;
    nodes[id].right = right;
    return id;
}

inline float half_area2(ez_vec3 aa, ez_vec3 bb) {  // "2.0 * (lx*ly + lx*lz + ly*lz)", :549
    float lenx = bb.x - aa.x, leny = bb.y - aa.y, lenz = bb.z - aa.z;
    return 2.0f * ((lenx * leny) + (lenx * lenz) + (leny * lenz));
}

// buildBVHwithSAH exactly as written, P5/main.cpp:458-589 (4 std::sorts of whole Triangles per node)
int build_sah_literal(std::vector<Tri>& tris, std::vector<Node>& nodes, int l, int r, int n) {
    if (l > r) return 0;
    nodes.push_back(Node());
    int id = (int)nodes.size() - 1;
    node_init(nodes[id]);
    for (int i = l; i <= r; i++) {
        nodes[id].AA = ez_vmin(nodes[id].AA, tri_min(tris[i]));
        nodes[id].BB = ez_vmax(nodes[id].BB, tri_max(tris[i]));
    }
    if ((r - l + 1) <= n) {
        nodes[id].n = r - l + 1;
        nodes[id].index = l;
        return id;
    }
    float Cost = EZ_INF;
    int Axis = 0;
    int Split = (l + r) / 2;
    for (int axis = 0; axis < 3; axis++) {
        if (axis == 0) std::sort(&tris[0] + l, &tris[0] + r + 1, cmpx);
        if (axis == 1) std::sort(&tris[0] + l, &tris[0] + r + 1, cmpy);
        if (axis == 2) std::sort(&tris[0] + l, &tris[0] + r + 1, cmpz);
        int cnt = r - l + 1;
        std::vector<ez_vec3> leftMax(cnt, ez_v3(-EZ_INF, -EZ_INF, -EZ_INF)), leftMin(cnt, ez_v3(EZ_INF, EZ_INF, EZ_INF));
        for (int i = l; i <= r; i++) {
            int bias = (i == l) ? 0 : 1;
            leftMax[i - l] = ez_vmax(leftMax[i - l - bias], tri_max(tris[i]));
            leftMin[i - l] = ez_vmin(leftMin[i - l - bias], tri_min(tris[i]));
        }
        std::vector<ez_vec3> rightMax(cnt, ez_v3(-EZ_INF, -EZ_INF, -EZ_INF)), rightMin(cnt, ez_v3(EZ_INF, EZ_INF, EZ_INF));
        for (int i = r; i >= l; i--) {
            int bias = (i == r) ? 0 : 1;
            rightMax[i - l] = ez_vmax(rightMax[i - l + bias], tri_max(tris[i]));
            rightMin[i - l] = ez_vmin(rightMin[i - l + bias], tri_min(tris[i]));
        }
        float cost = EZ_INF;
        int split = l;
        for (int i = l; i <= r - 1; i++) {
            float leftS = half_area2(leftMin[i - l], leftMax[i - l]);
            float leftCost = leftS * (float)(i - l + 1);
            float rightS = half_area2(rightMin[i + 1 - l], rightMax[i + 1 - l]);
            float rightCost = rightS * (float)(r - i);
            float totalCost = leftCost + rightCost;
            if (totalCost < cost) { cost = totalCost; split = i; }
        }
        if (cost < Cost) { Cost = cost; Axis = axis; Split = split; }
    }
    if (Axis == 0) std::sort(&tris[0] + l, &tris[0] + r + 1, cmpx);
    if (Axis == 1) std::sort(&tris[0] + l, &tris[0] + r + 1, cmpy);
    if (Axis == 2) std::sort(&tris[0] + l, &tris[0] + r + 1, cmpz);
    int left = build_sah_literal(tris, nodes, l, Split, n);
    int right = build_sah_literal(tris, nodes, Split + 1, r, n);
    nodes[id].left = left;
    nodes[id].right = right;
    return id;
}

// ---- fast builder: the same algorithm on 16-byte sort keys -------------------------------
// std::sort's control flow depends only on comparison outcomes, and the comparators below
// return exactly what cmpx/cmpy/cmpz return (the centroid is the same fp32 expression,
// evaluated once), so every std::sort call produces the permutation the literal builder
// produces; sub-trees are independent and are built on separate threads, then spliced in
// the literal builder's pre-order numbering.
struct Key {
    float cx, cy, cz;
    unsigned id;
};
struct FastCtx {
    const std::vector<ez_vec3>* bmin;
    const std::vector<ez_vec3>* bmax;
    Key* keys;
    int leaf_n;
    float inf;  // cost sentinel / box seed: EZ_INF (114514, the reference's quirk) or FLT_MAX (accel tree)
    int median_depth = 0;  // > 0 (acceleration tree only): below this depth split at the median, whatever the SAH says -- equal costs
                           // (coincident triangles) make the sweep peel one triangle per level, i.e. an O(n)-deep chain
};
bool kcmpx(const Key& a, const Key& b) { return a.cx < b.cx; }
bool kcmpy(const Key& a, const Key& b) { return a.cy < b.cy; }
bool kcmpz(const Key& a, const Key& b) { return a.cz < b.cz; }

// Appends the subtree for [l,r] to `out` in pre-order.  Child links are RELATIVE to the
// start of this subtree's block (0 = no child, as the root of a block is never a child).
void build_sah_fast(const FastCtx& cx, int l, int r, std::vector<Node>& out, int depth) {
    size_t base = out.size();
    out.push_back(Node());
    node_init(out[base]);
    Key* keys = cx.keys;
    const std::vector<ez_vec3>& bmin = *cx.bmin;
    const std::vector<ez_vec3>& bmax = *cx.bmax;
    {
        ez_vec3 AA = out[base].AA, BB = out[base].BB;
        for (int i = l; i <= r; i++) {
            AA = ez_vmin(AA, bmin[keys[i].id]);
            BB = ez_vmax(BB, bmax[keys[i].id]);
        }
        out[base].AA = AA;
        out[base].BB = BB;
    }
    int cnt = r - l + 1;
    if (cnt <= cx.leaf_n) {
        out[base].n = cnt;
        out[base].index = l;
        return;
    }
    const float INFV = cx.inf;
    float Cost = INFV;
    int Axis = 0;
    int Split = (l + r) / 2;
    {
        std::vector<ez_vec3> rightMax(cnt), rightMin(cnt);
        for (int axis = 0; axis < 3; axis++) {
            if (axis == 0) std::sort(keys + l, keys + r + 1, kcmpx);
            if (axis == 1) std::sort(keys + l, keys + r + 1, kcmpy);
            if (axis == 2) std::sort(keys + l, keys + r + 1, kcmpz);
            ez_vec3 rmax = ez_v3(-INFV, -INFV, -INFV), rmin = ez_v3(INFV, INFV, INFV);
            for (int i = r; i >= l; i--) {
                rmax = ez_vmax(rmax, bmax[keys[i].id]);
                rmin = ez_vmin(rmin, bmin[keys[i].id]);
                rightMax[i - l] = rmax;
                rightMin[i - l] = rmin;
            }
            float cost = INFV;
            int split = l;
            ez_vec3 lmax = ez_v3(-INFV, -INFV, -INFV), lmin = ez_v3(INFV, INFV, INFV);
            for (int i = l; i <= r - 1; i++) {
                lmax = ez_vmax(lmax, bmax[keys[i].id]);
                lmin = ez_vmin(lmin, bmin[keys[i].id]);
                float leftCost = half_area2(lmin, lmax) * (float)(i - l + 1);
                float rightCost = half_area2(rightMin[i + 1 - l], rightMax[i + 1 - l]) * (float)(r - i);
                float totalCost = leftCost + rightCost;
                if (totalCost < cost) { cost = totalCost; split = i; }
            }
            if (cost < Cost) { Cost = cost; Axis = axis; Split = split; }
        }
    }
    if (Axis == 0) std::sort(keys + l, keys + r + 1, kcmpx);
    if (Axis == 1) std::sort(keys + l, keys + r + 1, kcmpy);
    if (Axis == 2) std::sort(keys + l, keys + r + 1, kcmpz);
    if (cx.median_depth > 0 && depth >= cx.median_depth) Split = (l + r) / 2;

    std::vector<Node> leftNodes, rightNodes;
    bool par = (depth < 6) && (cnt > 4096);
    if (par) {
        auto fut = std::async(std::launch::async,
                              [&]() { build_sah_fast(cx, l, Split, leftNodes, depth + 1); });
        build_sah_fast(cx, Split + 1, r, rightNodes, depth + 1);
        fut.get();
    } else {
        build_sah_fast(cx, l, Split, leftNodes, depth + 1);
        build_sah_fast(cx, Split + 1, r, rightNodes, depth + 1);
    }
    // splice: [this][left block][right block]; links relative to `base`
    size_t lo = 1, ro = 1 + leftNodes.size();
    out[base].left = (int)lo;
    out[base].right = (int)ro;
    out.reserve(out.size() + leftNodes.size() + rightNodes.size());
    for (auto nd : leftNodes) {
        if (nd.left) nd.left += (int)lo;
        if (nd.right) nd.right += (int)lo;
        out.push_back(nd);
    }
    for (auto nd : rightNodes) {
        if (nd.left) nd.left += (int)ro;
        if (nd.right) nd.right += (int)ro;
        out.push_back(nd);
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------
struct ezrt_trilist {
    std::vector<Tri> tris;
    std::vector<Node> nodes;
};

// Acceleration tree for the device's default traversal policy (capi.cu): the same exhaustive-sweep
// SAH as buildBVHwithSAH but WITHOUT the reference's INF = 114514 cost sentinel, so the top levels
// are real SAH splits instead of median splits on axis 0.  nodes[0] is the root; child links are
// indices into `nodes` (0 = none); order[i] = index (in `tris`) of the i-th triangle of the tree.
// The sweep of buildBVHwithSAH re-sorts the node's triangles four times at every node (P5/main.cpp:493-575): O(n log^2 n),
// 1.4 s of the 1.7 s ezrt_scene_create took at 1 M triangles.  The acceleration tree does not have to reproduce the
// reference's permutation, so this builder sorts ONCE per axis and keeps the three orders through every split by stable
// partition (Wald 2007 "sort once"): the same cost function, the same exhaustive sweep over every split position of every
// axis, O(n log n).  Sub-trees are built on separate threads as in build_sah_fast.
namespace {
struct PresortCtx {
    const ez_vec3* bmin;
    const ez_vec3* bmax;
    uint32_t* idx[3];      // triangle ids of the whole array, three times: sorted by centroid x / y / z within every node's range
    uint32_t* tmp;         // partition scratch, n entries
    unsigned char* side;   // per triangle id: 1 = goes to the right child
    int leaf_n;
    int median_depth;
};

void build_accel_presorted(const PresortCtx& cx, int l, int r, std::vector<EzrtAccelNode>& out, int depth) {
    const size_t base = out.size();
    out.push_back(EzrtAccelNode());
    {
        ez_vec3 AA = ez_v3(3.0e38f, 3.0e38f, 3.0e38f), BB = ez_v3(-3.0e38f, -3.0e38f, -3.0e38f);
        const uint32_t* ix = cx.idx[0];
        for (int i = l; i <= r; i++) {
            AA = ez_vmin(AA, cx.bmin[ix[i]]);
            BB = ez_vmax(BB, cx.bmax[ix[i]]);
        }
        EzrtAccelNode& nd = out[base];
        nd.left = nd.right = nd.n = nd.index = 0;
        nd.AA[0] = AA.x; nd.AA[1] = AA.y; nd.AA[2] = AA.z;
        nd.BB[0] = BB.x; nd.BB[1] = BB.y; nd.BB[2] = BB.z;
    }
    const int cnt = r - l + 1;
    if (cnt <= cx.leaf_n) {
        out[base].n = cnt;
        out[base].index = l;
        return;
    }
    float Cost = 3.0e38f;
    int Axis = 0, Split = (l + r) / 2;
    {
        std::vector<float> rightArea(cnt);
        for (int axis = 0; axis < 3; axis++) {
            const uint32_t* ix = cx.idx[axis];
            ez_vec3 rmax = ez_v3(-3.0e38f, -3.0e38f, -3.0e38f), rmin = ez_v3(3.0e38f, 3.0e38f, 3.0e38f);
            for (int i = r; i > l; i--) {
                rmax = ez_vmax(rmax, cx.bmax[ix[i]]);
                rmin = ez_vmin(rmin, cx.bmin[ix[i]]);
                rightArea[i - l] = half_area2(rmin, rmax);
            }
            ez_vec3 lmax = ez_v3(-3.0e38f, -3.0e38f, -3.0e38f), lmin = ez_v3(3.0e38f, 3.0e38f, 3.0e38f);
            for (int i = l; i <= r - 1; i++) {
                lmax = ez_vmax(lmax, cx.bmax[ix[i]]);
                lmin = ez_vmin(lmin, cx.bmin[ix[i]]);
                const float total = half_area2(lmin, lmax) * (float)(i - l + 1) + rightArea[i + 1 - l] * (float)(r - i);
                if (total < Cost) { Cost = total; Axis = axis; Split = i; }
            }
        }
    }
    if (cx.median_depth > 0 && depth >= cx.median_depth) Split = (l + r) / 2;   // coincident triangles: no O(n)-deep chains
    // children keep the three orders: mark the sides along the split axis, stable-partition the other two
    for (int i = l; i <= r; i++) cx.side[cx.idx[Axis][i]] = (i > Split) ? 1 : 0;
    for (int a = 0; a < 3; a++) {
        if (a == Axis) continue;
        uint32_t* ix = cx.idx[a];
        int nl = l, nr = 0;
        for (int i = l; i <= r; i++) {
            const uint32_t t = ix[i];
            if (cx.side[t]) cx.tmp[l + nr++] = t; else ix[nl++] = t;
        }
        memcpy(ix + nl, cx.tmp + l, sizeof(uint32_t) * (size_t)nr);
    }
    std::vector<EzrtAccelNode> leftNodes, rightNodes;
    const bool par = (depth < 6) && (cnt > 4096);
    if (par) {
        auto fut = std::async(std::launch::async, [&]() { build_accel_presorted(cx, l, Split, leftNodes, depth + 1); });
        build_accel_presorted(cx, Split + 1, r, rightNodes, depth + 1);
        fut.get();
    } else {
        build_accel_presorted(cx, l, Split, leftNodes, depth + 1);
        build_accel_presorted(cx, Split + 1, r, rightNodes, depth + 1);
    }
    const int lo = 1, ro = 1 + (int)leftNodes.size();   // splice: [this][left block][right block], links relative to this block
    out[base].left = lo;
    out[base].right = ro;
    out.reserve(out.size() + leftNodes.size() + rightNodes.size());
    for (auto nd : leftNodes) {
        if (nd.n <= 0) { nd.left += lo; nd.right += lo; }
        out.push_back(nd);
    }
    for (auto nd : rightNodes) {
        if (nd.n <= 0) { nd.left += ro; nd.right += ro; }
        out.push_back(nd);
    }
}
}  // namespace

int ezrt_build_accel(const float* tris, int n_tris, int leaf_n, std::vector<EzrtAccelNode>& nodes_out, std::vector<uint32_t>& order) {
    std::vector<ez_vec3> bmin(n_tris), bmax(n_tris), cen(n_tris);
    for (int i = 0; i < n_tris; i++) {
        const float* t = tris + (size_t)i * EZRT_TRIANGLE_FLOATS;
        Tri tr;
        tr.p1 = ez_v3(t[0], t[1], t[2]); tr.p2 = ez_v3(t[3], t[4], t[5]); tr.p3 = ez_v3(t[6], t[7], t[8]);
        cen[i] = centroid(tr);
        bmin[i] = tri_min(tr);
        bmax[i] = tri_max(tr);
    }
    std::vector<uint32_t> idx[3], tmp(n_tris);
    std::vector<unsigned char> side(n_tris, 0);
    {
        std::future<void> f[3];
        for (int a = 0; a < 3; a++) {
            idx[a].resize(n_tris);
            for (int i = 0; i < n_tris; i++) idx[a][i] = (uint32_t)i;
            f[a] = std::async(std::launch::async, [&, a]() {
                const ez_vec3* c = cen.data();
                if (a == 0) std::stable_sort(idx[0].begin(), idx[0].end(), [c](uint32_t p, uint32_t q) { return c[p].x < c[q].x; });
                if (a == 1) std::stable_sort(idx[1].begin(), idx[1].end(), [c](uint32_t p, uint32_t q) { return c[p].y < c[q].y; });
                if (a == 2) std::stable_sort(idx[2].begin(), idx[2].end(), [c](uint32_t p, uint32_t q) { return c[p].z < c[q].z; });
            });
        }
        for (int a = 0; a < 3; a++) f[a].get();
    }
    PresortCtx cx;
    cx.bmin = bmin.data(); cx.bmax = bmax.data();
    cx.idx[0] = idx[0].data(); cx.idx[1] = idx[1].data(); cx.idx[2] = idx[2].data();
    cx.tmp = tmp.data(); cx.side = side.data();
    cx.leaf_n = leaf_n;
    cx.median_depth = 32;   // depth <= 32 + log2(n): the traversal stacks always suffice, the recursion stays shallow
    nodes_out.clear();
    build_accel_presorted(cx, 0, n_tris - 1, nodes_out, 0);
    order = idx[0];
    return (int)nodes_out.size();
}

extern "C" {

ezrt_trilist* ezrt_trilist_create(void) { return new (std::nothrow) ezrt_trilist(); }
void ezrt_trilist_destroy(ezrt_trilist* list) { delete list; }
int ezrt_trilist_size(const ezrt_trilist* list) { return list ? (int)list->tris.size() : EZRT_ERR_INVALID; }
int ezrt_trilist_node_count(const ezrt_trilist* list) { return list ? (int)list->nodes.size() : EZRT_ERR_INVALID; }

void ezrt_transform_matrix(const float rotate_deg[3], const float translate[3], const float scale[3], float out[16]) {
    Mat4 m = transform_matrix(rotate_deg, translate, scale);
    memcpy(out, m.c, sizeof(float) * 16);
}

int ezrt_trilist_read_obj(ezrt_trilist* list, const char* path, const float material[EZRT_MATERIAL_FLOATS],
                          const float trans[16], int smooth_normal) {
    if (!list || !path || !material || !trans) return ezrt_set_error(EZRT_ERR_INVALID, "read_obj: null argument");
    std::ifstream fin(path);
    if (!fin.is_open()) return ezrt_set_error(EZRT_ERR_IO, "read_obj: cannot open %s", path);
    Mat4 m;
    memcpy(m.c, trans, sizeof(float) * 16);
    int rc = read_obj_stream(fin, list->tris, material, m, (smooth_normal & 1) != 0, (smooth_normal & EZRT_OBJ_HARDENED) != 0);
    if (rc) return ezrt_set_error(rc, "read_obj: malformed face in %s", path);
    return EZRT_OK;
}

int ezrt_trilist_read_obj_text(ezrt_trilist* list, const char* text, size_t len,
                               const float material[EZRT_MATERIAL_FLOATS], const float trans[16], int smooth_normal) {
    if (!list || !text || !material || !trans) return ezrt_set_error(EZRT_ERR_INVALID, "read_obj_text: null argument");
    std::istringstream fin(std::string(text, len));
    Mat4 m;
    memcpy(m.c, trans, sizeof(float) * 16);
    int rc = read_obj_stream(fin, list->tris, material, m, (smooth_normal & 1) != 0, (smooth_normal & EZRT_OBJ_HARDENED) != 0);
    if (rc) return ezrt_set_error(rc, "read_obj_text: malformed face");
    return EZRT_OK;
}

int ezrt_trilist_read_obj_textured(ezrt_trilist* list, const char* path, const float material[EZRT_MATERIAL_FLOATS],
                                   const float trans[16], int smooth_normal, int32_t texture_id) {
    if (!list || !path || !material || !trans || texture_id < -1) return ezrt_set_error(EZRT_ERR_INVALID, "read_obj_textured: bad argument");
    std::ifstream fin(path);
    if (!fin.is_open()) return ezrt_set_error(EZRT_ERR_IO, "read_obj_textured: cannot open %s", path);
    Mat4 m;
    memcpy(m.c, trans, sizeof(float) * 16);
    int rc = read_obj_stream(fin, list->tris, material, m, (smooth_normal & 1) != 0, (smooth_normal & EZRT_OBJ_HARDENED) != 0, true, texture_id);
    if (rc) return ezrt_set_error(rc, "read_obj_textured: malformed face or texture index in %s", path);
    return EZRT_OK;
}

int ezrt_trilist_read_obj_textured_text(ezrt_trilist* list, const char* text, size_t len, const float material[EZRT_MATERIAL_FLOATS],
                                        const float trans[16], int smooth_normal, int32_t texture_id) {
    if (!list || !text || !material || !trans || texture_id < -1) return ezrt_set_error(EZRT_ERR_INVALID, "read_obj_textured_text: bad argument");
    std::istringstream fin(std::string(text, len));
    Mat4 m;
    memcpy(m.c, trans, sizeof(float) * 16);
    int rc = read_obj_stream(fin, list->tris, material, m, (smooth_normal & 1) != 0, (smooth_normal & EZRT_OBJ_HARDENED) != 0, true, texture_id);
    if (rc) return ezrt_set_error(rc, "read_obj_textured_text: malformed face or texture index");
    return EZRT_OK;
}

int ezrt_trilist_encode_texcoords(const ezrt_trilist* list, float* uv_out, int32_t* id_out) {
    if (!list || !uv_out || !id_out) return ezrt_set_error(EZRT_ERR_INVALID, "encode_texcoords: null argument");
    for (size_t i = 0; i < list->tris.size(); i++) {
        memcpy(uv_out + 6 * i, list->tris[i].uv, sizeof(float) * 6);
        id_out[i] = list->tris[i].tex_id;
    }
    return EZRT_OK;
}

int ezrt_trilist_append_encoded(ezrt_trilist* list, const float* tris, int n) {
    if (!list || (!tris && n > 0) || n < 0) return ezrt_set_error(EZRT_ERR_INVALID, "append_encoded: bad argument");
    size_t off = list->tris.size();
    list->tris.resize(off + (size_t)n);
    for (int i = 0; i < n; i++) {
        const float* s = tris + (size_t)i * EZRT_TRIANGLE_FLOATS;
        Tri& t = list->tris[off + i];
        t.p1 = ez_v3(s[0], s[1], s[2]);   t.p2 = ez_v3(s[3], s[4], s[5]);   t.p3 = ez_v3(s[6], s[7], s[8]);
        t.n1 = ez_v3(s[9], s[10], s[11]); t.n2 = ez_v3(s[12], s[13], s[14]); t.n3 = ez_v3(s[15], s[16], s[17]);
        memcpy(t.material, s + 18, sizeof(float) * EZRT_MATERIAL_FLOATS);
    }
    return EZRT_OK;
}

// The reference sorts triangles with std::sort and an order-only comparator (P5/main.cpp:395-455, :458-589): which of several
// triangles with EQUAL centroid coordinates ends up where is a property of the C++ library's introsort, and the triangle order
// decides the tree and (through leaf order and ties) the image.  The goldens of this repository and the reference's own uploads
// (tests/test_ref_host.py) were produced with libstdc++.  This known-answer check sorts a fixed array with many equal keys and
// compares the permutation with libstdc++'s; a host whose std::sort differs still builds a VALID tree, but not the reference's.
static uint32_t sort_kat_hash() {
    struct E { int key, id; };
    std::vector<E> v(613);
    uint32_t x = 2463534242u;
    for (int i = 0; i < (int)v.size(); i++) {
        x ^= x << 13; x ^= x >> 17; x ^= x << 5;
        v[i].key = (int)(x % 23u);
        v[i].id = i;
    }
    std::sort(v.begin(), v.end(), [](const E& a, const E& b) { return a.key < b.key; });
    uint32_t h = 2166136261u;
    for (const E& e : v) h = (h ^ (uint32_t)e.id) * 16777619u;
    return h;
}
#define EZRT_SORT_KAT_LIBSTDCXX 1126591013u

int ezrt_host_sort_is_reference(void) { return sort_kat_hash() == EZRT_SORT_KAT_LIBSTDCXX ? 1 : 0; }

int ezrt_trilist_build_bvh(ezrt_trilist* list, int leaf_n, int builder) {
    {
        static int warned = 0;
        if (!warned && builder != EZRT_BVH_SAH_NO_SENTINEL && !ezrt_host_sort_is_reference()) {
            warned = 1;
            fprintf(stderr, "ezrt: this C++ library's std::sort orders equal keys differently from libstdc++: the BVH is valid but is not "
                            "the reference's triangle order (ezrt_host_sort_is_reference() == 0)\n");
        }
    }
    if (!list || leaf_n < 1) return ezrt_set_error(EZRT_ERR_INVALID, "build_bvh: bad argument");
    if (list->tris.empty()) return ezrt_set_error(EZRT_ERR_INVALID, "build_bvh: empty triangle list");
    // nodes{testNode}: the recognisable dummy element 0 (P5/main.cpp:830-836)
    Node testNode;
    testNode.left = 255; testNode.right = 128; testNode.n = 30; testNode.index = 0;
    testNode.AA = ez_v3(1, 1, 0);
    testNode.BB = ez_v3(0, 1, 0);
    list->nodes.clear();
    list->nodes.push_back(testNode);
    int N = (int)list->tris.size();
    if (builder == EZRT_BVH_SAH_LITERAL) {
        build_sah_literal(list->tris, list->nodes, 0, N - 1, leaf_n);
    } else if (builder == EZRT_BVH_MEDIAN) {
        build_median(list->tris, list->nodes, 0, N - 1, leaf_n);
    } else if (builder == EZRT_BVH_SAH_FAST || builder == EZRT_BVH_SAH_NO_SENTINEL) {
        std::vector<Key> keys(N);
        std::vector<ez_vec3> bmin(N), bmax(N);
        for (int i = 0; i < N; i++) {
            ez_vec3 c = centroid(list->tris[i]);
            keys[i].cx = c.x; keys[i].cy = c.y; keys[i].cz = c.z; keys[i].id = (unsigned)i;
            bmin[i] = tri_min(list->tris[i]);
            bmax[i] = tri_max(list->tris[i]);
        }
        FastCtx cx;
        cx.bmin = &bmin; cx.bmax = &bmax; cx.keys = keys.data(); cx.leaf_n = leaf_n;
        cx.inf = (builder == EZRT_BVH_SAH_NO_SENTINEL) ? 3.0e38f : EZ_INF;
        std::vector<Node> sub;
        build_sah_fast(cx, 0, N - 1, sub, 0);
        for (auto nd : sub) {  // relative-to-block-0 -> absolute (dummy node shifts everything by 1)
            if (nd.left) nd.left += 1;
            if (nd.right) nd.right += 1;
            list->nodes.push_back(nd);
        }
        std::vector<Tri> sorted(N);
        for (int i = 0; i < N; i++) sorted[i] = list->tris[keys[i].id];
        list->tris.swap(sorted);
    } else {
        return ezrt_set_error(EZRT_ERR_INVALID, "build_bvh: unknown builder %d", builder);
    }
    return (int)list->nodes.size();
}

int ezrt_trilist_encode_triangles(const ezrt_trilist* list, float* out) {
    if (!list || !out) return ezrt_set_error(EZRT_ERR_INVALID, "encode_triangles: null argument");
    for (size_t i = 0; i < list->tris.size(); i++) {
        const Tri& t = list->tris[i];
        float* d = out + i * EZRT_TRIANGLE_FLOATS;
        d[0] = t.p1.x; d[1] = t.p1.y; d[2] = t.p1.z;
        d[3] = t.p2.x; d[4] = t.p2.y; d[5] = t.p2.z;
        d[6] = t.p3.x; d[7] = t.p3.y; d[8] = t.p3.z;
        d[9] = t.n1.x; d[10] = t.n1.y; d[11] = t.n1.z;
        d[12] = t.n2.x; d[13] = t.n2.y; d[14] = t.n2.z;
        d[15] = t.n3.x; d[16] = t.n3.y; d[17] = t.n3.z;
        // emissive, baseColor, param1..param4 = the Material in declaration order (P5/main.cpp:856-861)
        memcpy(d + 18, t.material, sizeof(float) * EZRT_MATERIAL_FLOATS);
    }
    return EZRT_OK;
}

int ezrt_trilist_encode_nodes(const ezrt_trilist* list, float* out) {
    if (!list || !out) return ezrt_set_error(EZRT_ERR_INVALID, "encode_nodes: null argument");
    for (size_t i = 0; i < list->nodes.size(); i++) {
        const Node& nd = list->nodes[i];
        float* d = out + i * EZRT_BVHNODE_FLOATS;
        d[0] = (float)nd.left; d[1] = (float)nd.right; d[2] = 0.0f;
        d[3] = (float)nd.n; d[4] = (float)nd.index; d[5] = 0.0f;
        d[6] = nd.AA.x; d[7] = nd.AA.y; d[8] = nd.AA.z;
        d[9] = nd.BB.x; d[10] = nd.BB.y; d[11] = nd.BB.z;
    }
    return EZRT_OK;
}

// ---- HDRLoader::load, P5/lib/hdrloader.cpp:29-97 (RLE + flat RGBE scanlines) --------------
namespace {
typedef unsigned char RGBE[4];

// Hardened against what the reference's decoder trusts the file for (hdrloader.cpp:161-191): a run marker (1,1,1,n) needs
// a previous pixel IN THIS SCANLINE to repeat (the reference reads scanline[-1], i.e. before the buffer, for a marker at
// x = 0), and the run length n << rshift must stay defined (rshift = 32 after four consecutive markers is UB in C).
bool old_decrunch(RGBE* scanline, int len, FILE* file, const RGBE* line_start) {
    int rshift = 0;
    while (len > 0) {
        scanline[0][0] = (unsigned char)fgetc(file);
        scanline[0][1] = (unsigned char)fgetc(file);
        scanline[0][2] = (unsigned char)fgetc(file);
        scanline[0][3] = (unsigned char)fgetc(file);
        if (feof(file)) return false;
        if (scanline[0][0] == 1 && scanline[0][1] == 1 && scanline[0][2] == 1) {
            if (scanline == line_start || rshift > 24) return false;   // malformed: nothing to repeat / run length overflow
            for (int i = scanline[0][3] << rshift; i > 0 && len > 0; i--) {
                memcpy(&scanline[0][0], &scanline[-1][0], 4);
                scanline++;
                len--;
            }
            rshift += 8;
        } else {
            scanline++;
            len--;
            rshift = 0;
        }
    }
    return true;
}

bool decrunch(RGBE* scanline, int len, FILE* file) {  // hdrloader.cpp:118-159
    if (len < 8 || len > 0x7fff) return old_decrunch(scanline, len, file, scanline);
    int i = fgetc(file);
    if (i != 2) {
        fseek(file, -1, SEEK_CUR);
        return old_decrunch(scanline, len, file, scanline);
    }
    scanline[0][1] = (unsigned char)fgetc(file);
    scanline[0][2] = (unsigned char)fgetc(file);
    i = fgetc(file);
    if (scanline[0][1] != 2 || (scanline[0][2] & 128)) {
        scanline[0][0] = 2;
        scanline[0][3] = (unsigned char)i;
        return old_decrunch(scanline + 1, len - 1, file, scanline);
    }
    for (i = 0; i < 4; i++) {
        for (int j = 0; j < len;) {
            unsigned char code = (unsigned char)fgetc(file);
            if (feof(file)) return false;
            if (code > 128) {
                code &= 127;
                unsigned char val = (unsigned char)fgetc(file);
                while (code-- && j < len) scanline[j++][i] = val;
            } else {
                while (code-- && j < len) scanline[j++][i] = (unsigned char)fgetc(file);
            }
        }
    }
    return feof(file) ? false : true;
}

inline float convert_component(int expo, int val) {  // hdrloader.cpp:99-104: (val/256) * 2^expo, exact
    float v = (float)val / 256.0f;
    return ez_ldexp(v, expo);
}
}  // namespace

int ezrt_hdr_load(const char* path, int* width, int* height, float* cols) {
    if (!path || !width || !height) return ezrt_set_error(EZRT_ERR_INVALID, "hdr_load: null argument");
    FILE* file = fopen(path, "rb");
    if (!file) return ezrt_set_error(EZRT_ERR_IO, "hdr_load: cannot open %s", path);
    char str[16];
    if (fread(str, 10, 1, file) != 1 || memcmp(str, "#?RADIANCE", 10)) {
        fclose(file);
        return ezrt_set_error(EZRT_ERR_IO, "hdr_load: %s is not a Radiance file", path);
    }
    fseek(file, 1, SEEK_CUR);
    int c = 0, oldc;
    while (true) {  // header commands end with an empty line
        oldc = c;
        c = fgetc(file);
        if (c == EOF) { fclose(file); return ezrt_set_error(EZRT_ERR_IO, "hdr_load: truncated header"); }
        if (c == 0xa && oldc == 0xa) break;
    }
    char reso[200];
    int i = 0;
    while (i < 199) {
        c = fgetc(file);
        if (c == EOF) break;
        reso[i++] = (char)c;
        if (c == 0xa) break;
    }
    reso[i] = 0;
    int w = 0, h = 0;
    if (sscanf(reso, "-Y %d +X %d", &h, &w) != 2 || w <= 0 || h <= 0) {  // "%ld" into int in the reference (UB on LP64)
        fclose(file);
        return ezrt_set_error(EZRT_ERR_IO, "hdr_load: unsupported resolution line");
    }
    *width = w;
    *height = h;
    if (!cols) { fclose(file); return EZRT_OK; }
    std::vector<unsigned char> buf((size_t)w * 4);
    RGBE* scanline = reinterpret_cast<RGBE*>(buf.data());
    memset(cols, 0, sizeof(float) * (size_t)w * h * 3);
    float* out = cols;
    bool truncated = false;
    for (int y = h - 1; y >= 0; y--) {
        if (!decrunch(scanline, w, file)) { truncated = true; break; }  // the reference stops here too and keeps what it has (rows of 0)
        for (int x = 0; x < w; x++) {  // workOnRGBE, hdrloader.cpp:106-116
            int expo = (int)scanline[x][3] - 128;
            out[0] = convert_component(expo, scanline[x][0]);
            out[1] = convert_component(expo, scanline[x][1]);
            out[2] = convert_component(expo, scanline[x][2]);
            out += 3;
        }
    }
    fclose(file);
    return truncated ? 1 : EZRT_OK;   // 1: the pixel data ended early or was malformed; the remaining rows are zero (include/ezrt.h)
}

// ---- calculateHdrCache, P5/main.cpp:592-689 ------------------------------------------------
int ezrt_hdr_cache(const float* HDR, int width, int height, float* cache) {
    if (!HDR || !cache || width <= 0 || height <= 0) return ezrt_set_error(EZRT_ERR_INVALID, "hdr_cache: bad argument");
    const size_t W = (size_t)width, H = (size_t)height;
    std::vector<float> pdf(W * H);
    float lumSum = 0.0f;
    for (size_t i = 0; i < H; i++)
        for (size_t j = 0; j < W; j++) {
            float R = HDR[3 * (i * W + j)], G = HDR[3 * (i * W + j) + 1], B = HDR[3 * (i * W + j) + 2];
            float lum = (float)((0.2 * (double)R + 0.7 * (double)G) + 0.1 * (double)B);  // :604 -- the literals are doubles
            pdf[i * W + j] = lum;
            lumSum += lum;
        }
    for (size_t k = 0; k < W * H; k++) pdf[k] /= lumSum;
    std::vector<float> pdf_x_margin(W, 0.0f);
    for (size_t j = 0; j < W; j++)
        for (size_t i = 0; i < H; i++) pdf_x_margin[j] += pdf[i * W + j];
    std::vector<float> cdf_x_margin = pdf_x_margin;
    for (size_t i = 1; i < W; i++) cdf_x_margin[i] += cdf_x_margin[i - 1];
    // conditional cdf of y given X=x, stored column-major: cdf_y[j*H + i]
    std::vector<float> cdf_y(W * H);
    for (size_t j = 0; j < W; j++) {
        float acc = 0.0f;
        for (size_t i = 0; i < H; i++) {
            float p = pdf[i * W + j] / pdf_x_margin[j];
            acc = (i == 0) ? p : (p + acc);  // cdf[i] += cdf[i-1]  ==  pdf_cond[i] + cdf[i-1]
            cdf_y[j * H + i] = acc;
        }
    }
    for (size_t j = 0; j < W; j++)
        for (size_t i = 0; i < H; i++) {
            float xi_1 = (float)i / (float)height;
            float xi_2 = (float)j / (float)width;
            size_t x = std::lower_bound(cdf_x_margin.begin(), cdf_x_margin.end(), xi_1) - cdf_x_margin.begin();
            if (x >= W) x = W - 1;  // the reference indexes out of bounds here; clamp
            const float* col = &cdf_y[x * H];
            size_t y = std::lower_bound(col, col + H, xi_2) - col;
            cache[3 * (i * W + j)] = (float)x / (float)width;
            cache[3 * (i * W + j) + 1] = (float)y / (float)height;
            cache[3 * (i * W + j) + 2] = pdf[i * W + j];
        }
    return EZRT_OK;
}

// ---- scene description file (SURVEY.md 8f row 4): replaces the hard-coded scene blocks of main()
// (P3/main.cpp:688-701, P4/main.cpp:687-729, P5/main.cpp:795-823).  Line oriented, '#' comments:
//   set <field> <values...>   field of the current Material (emissive, baseColor: 3 floats; others: 1)
//   reset                     back to the reference's default Material (P5/main.cpp:27-42)
//   mesh <obj path> smooth|flat [hardened] rotate rx ry rz translate tx ty tz scale sx sy sz
//   camera <rotatAngle> <upAngle> <r>          (P5/main.cpp:796-798)
//   hdr <path>
// Relative paths are resolved against the scene file's directory.
int ezrt_scene_file_load(const char* path, ezrt_trilist* list, float camera[3], char* hdr_path, size_t hdr_path_cap) {
    if (!path || !list) return ezrt_set_error(EZRT_ERR_INVALID, "scene_file_load: null argument");
    std::ifstream fin(path);
    if (!fin.is_open()) return ezrt_set_error(EZRT_ERR_IO, "scene_file_load: cannot open %s", path);
    std::string dir(path);
    size_t slash = dir.find_last_of('/');
    dir = (slash == std::string::npos) ? std::string() : dir.substr(0, slash + 1);
    auto resolve = [&](const std::string& p) { return (!p.empty() && p[0] == '/') ? p : dir + p; };
    const float defaults[EZRT_MATERIAL_FLOATS] = {0, 0, 0, 1, 1, 1, 0.0f, 0.0f, 0.5f, 0.0f, 0.5f, 0.0f, 0.0f, 0.5f, 0.0f, 1.0f, 1.0f, 0.0f};
    float mat[EZRT_MATERIAL_FLOATS];
    memcpy(mat, defaults, sizeof(mat));
    static const char* names[] = {"subsurface", "metallic", "specular", "specularTint", "roughness", "anisotropic", "sheen", "sheenTint",
                                  "clearcoat", "clearcoatGloss", "IOR", "transmission"};
    if (camera) { camera[0] = 0.0f; camera[1] = 0.0f; camera[2] = 4.0f; }  // rotatAngle, upAngle, r defaults (P5/main.cpp:149-151)
    if (hdr_path && hdr_path_cap) hdr_path[0] = 0;
    std::string line;
    int lineno = 0;
    while (std::getline(fin, line)) {
        lineno++;
        size_t hash = line.find('#');
        if (hash != std::string::npos) line = line.substr(0, hash);
        std::istringstream sin(line);
        std::string cmd;
        if (!(sin >> cmd)) continue;
        if (cmd == "reset") {
            memcpy(mat, defaults, sizeof(mat));
        } else if (cmd == "set") {
            std::string field;
            sin >> field;
            if (field == "emissive" || field == "baseColor") {
                float* dst = mat + (field == "emissive" ? 0 : 3);
                if (!(sin >> dst[0] >> dst[1] >> dst[2])) return ezrt_set_error(EZRT_ERR_IO, "%s:%d: set %s needs 3 numbers", path, lineno, field.c_str());
            } else {
                int k = -1;
                for (int i = 0; i < 12; i++)
                    if (field == names[i]) k = i;
                if (k < 0 || !(sin >> mat[6 + k])) return ezrt_set_error(EZRT_ERR_IO, "%s:%d: bad material field '%s'", path, lineno, field.c_str());
            }
        } else if (cmd == "mesh") {
            std::string file, mode, key;
            if (!(sin >> file >> mode) || (mode != "smooth" && mode != "flat")) return ezrt_set_error(EZRT_ERR_IO, "%s:%d: mesh <path> smooth|flat ...", path, lineno);
            float rot[3] = {0, 0, 0}, tr[3] = {0, 0, 0}, sc[3] = {1, 1, 1};
            int flags = (mode == "smooth") ? 1 : 0;
            while (sin >> key) {
                float* dst = (key == "rotate") ? rot : (key == "translate") ? tr : (key == "scale") ? sc : nullptr;
                if (key == "hardened") { flags |= EZRT_OBJ_HARDENED; continue; }
                if (!dst || !(sin >> dst[0] >> dst[1] >> dst[2])) return ezrt_set_error(EZRT_ERR_IO, "%s:%d: bad mesh option '%s'", path, lineno, key.c_str());
            }
            float m16[16];
            ezrt_transform_matrix(rot, tr, sc, m16);
            int rc = ezrt_trilist_read_obj(list, resolve(file).c_str(), mat, m16, flags);
            if (rc) return rc;
        } else if (cmd == "camera") {
            float c[3];
            if (!(sin >> c[0] >> c[1] >> c[2])) return ezrt_set_error(EZRT_ERR_IO, "%s:%d: camera <rotatAngle> <upAngle> <r>", path, lineno);
            if (camera) memcpy(camera, c, sizeof(c));
        } else if (cmd == "hdr") {
            std::string file;
            if (!(sin >> file)) return ezrt_set_error(EZRT_ERR_IO, "%s:%d: hdr <path>", path, lineno);
            std::string full = resolve(file);
            if (hdr_path && hdr_path_cap) {
                if (full.size() + 1 > hdr_path_cap) return ezrt_set_error(EZRT_ERR_INVALID, "%s:%d: hdr path too long", path, lineno);
                memcpy(hdr_path, full.c_str(), full.size() + 1);
            }
        } else {
            return ezrt_set_error(EZRT_ERR_IO, "%s:%d: unknown directive '%s'", path, lineno, cmd.c_str());
        }
    }
    return EZRT_OK;
}

// ---- PNG output (role of P1's imshow + svpng, P1/main.cpp:173-194): 8-bit RGB, zlib "stored" blocks --
namespace {
struct PngOut {
    FILE* f;
    uint32_t crc;
    void raw(const unsigned char* p, size_t n) { fwrite(p, 1, n, f); }
    void u32(uint32_t v) { unsigned char b[4] = {(unsigned char)(v >> 24), (unsigned char)(v >> 16), (unsigned char)(v >> 8), (unsigned char)v}; raw(b, 4); }
    void crc_bytes(const unsigned char* p, size_t n) {
        static uint32_t table[256];
        static bool init = false;
        if (!init) {
            for (uint32_t i = 0; i < 256; i++) {
                uint32_t c = i;
                for (int k = 0; k < 8; k++) c = (c & 1u) ? (0xEDB88320u ^ (c >> 1)) : (c >> 1);
                table[i] = c;
            }
            init = true;
        }
        for (size_t i = 0; i < n; i++) crc = table[(crc ^ p[i]) & 0xffu] ^ (crc >> 8);
    }
    void chunk(const char* tag, const std::vector<unsigned char>& data) {
        u32((uint32_t)data.size());
        crc = 0xffffffffu;
        crc_bytes((const unsigned char*)tag, 4);
        raw((const unsigned char*)tag, 4);
        if (!data.empty()) { crc_bytes(data.data(), data.size()); raw(data.data(), data.size()); }
        u32(crc ^ 0xffffffffu);
    }
};
}  // namespace

int ezrt_write_png(const char* path, const float* fb, int width, int height, int channels, int tonemap) {
    if (!path || !fb || width <= 0 || height <= 0 || (channels != 3 && channels != 4)) return ezrt_set_error(EZRT_ERR_INVALID, "write_png: bad argument");
    // scanlines top row first (framebuffer row 0 is the bottom row), filter byte 0, quantised as imshow()
    const size_t stride = (size_t)width * 3 + 1;
    std::vector<unsigned char> rawimg(stride * height);
    for (int y = 0; y < height; y++) {
        unsigned char* row = &rawimg[(size_t)y * stride];
        row[0] = 0;
        const float* src = fb + (size_t)(height - 1 - y) * width * channels;
        for (int x = 0; x < width; x++) {
            ez_vec3 c = ez_v3(src[(size_t)x * channels], src[(size_t)x * channels + 1], src[(size_t)x * channels + 2]);
            if (tonemap) c = ez_tonemap_pass3(c, 1.5f);
            const float v[3] = {c.x, c.y, c.z};
            for (int k = 0; k < 3; k++) {
                float q = v[k] * 255.0f;
                q = (q != q) ? 0.0f : ez_min(ez_max(q, 0.0f), 255.0f);
                row[1 + 3 * x + k] = (unsigned char)q;
            }
        }
    }
    std::vector<unsigned char> z;
    z.push_back(0x78); z.push_back(0x01);  // zlib header, no compression
    uint32_t a = 1, b = 0;                 // adler32
    for (unsigned char c : rawimg) { a = (a + c) % 65521u; b = (b + a) % 65521u; }
    size_t pos = 0;
    while (pos < rawimg.size()) {
        size_t n = std::min<size_t>(65535, rawimg.size() - pos);
        z.push_back(pos + n == rawimg.size() ? 1 : 0);
        z.push_back((unsigned char)(n & 0xff)); z.push_back((unsigned char)(n >> 8));
        z.push_back((unsigned char)(~n & 0xff)); z.push_back((unsigned char)((~n >> 8) & 0xff));
        z.insert(z.end(), rawimg.begin() + pos, rawimg.begin() + pos + n);
        pos += n;
    }
    const uint32_t adler = (b << 16) | a;
    z.push_back((unsigned char)(adler >> 24)); z.push_back((unsigned char)(adler >> 16)); z.push_back((unsigned char)(adler >> 8)); z.push_back((unsigned char)adler);
    FILE* f = fopen(path, "wb");
    if (!f) return ezrt_set_error(EZRT_ERR_IO, "write_png: cannot open %s", path);
    PngOut out{f, 0};
    const unsigned char sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
    out.raw(sig, 8);
    std::vector<unsigned char> ihdr = {(unsigned char)(width >> 24), (unsigned char)(width >> 16), (unsigned char)(width >> 8), (unsigned char)width,
                                       (unsigned char)(height >> 24), (unsigned char)(height >> 16), (unsigned char)(height >> 8), (unsigned char)height,
                                       8, 2, 0, 0, 0};
    out.chunk("IHDR", ihdr);
    out.chunk("IDAT", z);
    out.chunk("IEND", std::vector<unsigned char>());
    fclose(f);
    return EZRT_OK;
}

// ---- display() camera, P5/main.cpp:710-713 -------------------------------------------------
void ezrt_camera_orbit(float rotatAngle, float upAngle, float r, float eye_out[3], float camera_rotate[16]) {
    float ra = rotatAngle * kDegToRad, ua = upAngle * kDegToRad;
    ez_vec3 eye = ez_v3(-ez_sin(ra) * ez_cos(ua), ez_sin(ua), ez_cos(ra) * ez_cos(ua));
    eye.x *= r; eye.y *= r; eye.z *= r;
    Mat4 look = mat_look_at(eye, ez_v3(0, 0, 0), ez_v3(0, 1, 0));
    Mat4 inv = mat_inverse(look);
    eye_out[0] = eye.x; eye_out[1] = eye.y; eye_out[2] = eye.z;
    memcpy(camera_rotate, inv.c, sizeof(float) * 16);
}

// ---- look-at camera with field of view and aspect: inverse(lookAt) has columns (s, u, -f, eye) (mat_look_at's basis)
int ezrt_camera_look_at(const float eye[3], const float target[3], const float up[3], float vfov_deg, float aspect, float cam_out[16]) {
    if (!eye || !target || !up || !cam_out) return ezrt_set_error(EZRT_ERR_INVALID, "camera_look_at: null argument");
    if (!(vfov_deg > 0.0f && vfov_deg < 180.0f) || !(aspect > 0.0f) || !ez_finite(aspect))
        return ezrt_set_error(EZRT_ERR_INVALID, "camera_look_at: need 0 < vfov_deg < 180 and a finite aspect > 0");
    const ez_vec3 e = ez_v3(eye[0], eye[1], eye[2]);
    const ez_vec3 d = ez_sub(ez_v3(target[0], target[1], target[2]), e);
    const ez_vec3 c = ez_cross(ez_normalize(d), ez_v3(up[0], up[1], up[2]));
    const float dd = ez_dot(d, d), cc = ez_dot(c, c);
    if (!(dd > 0.0f) || !ez_finite(dd) || !(cc > 0.0f) || !ez_finite(cc) || !ez_finite(e.x) || !ez_finite(e.y) || !ez_finite(e.z))
        return ezrt_set_error(EZRT_ERR_INVALID, "camera_look_at: degenerate view (eye == target, up parallel to the view, or not finite)");
    const ez_vec3 f = ez_normalize(d);
    const ez_vec3 s = ez_normalize(ez_cross(f, ez_v3(up[0], up[1], up[2])));
    const ez_vec3 u = ez_cross(s, f);
    const double t = tan(0.5 * (double)vfov_deg * 0.017453292519943295769);
    const float sy = (float)(t * 1.5), sx = (float)((double)aspect * t * 1.5);
    const float m[16] = {s.x * sx, s.y * sx, s.z * sx, 0.0f, u.x * sy, u.y * sy, u.z * sy, 0.0f, -f.x, -f.y, -f.z, 0.0f, e.x, e.y, e.z, 1.0f};
    memcpy(cam_out, m, sizeof(m));
    return EZRT_OK;
}

}  // extern "C"
