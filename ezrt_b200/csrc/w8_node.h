// w8_node.h -- the 8-wide, 8-bit-quantised node of the device's acceleration tree (DESIGN.md section 4, "W8").
// Shared by the host builder (accel_w8.cpp), the kernels (device_functions.cuh) and the CPU model of the
// traversal (tools/w8_model.cpp), so that all three use the same layout and the same decode arithmetic.
//
// The reference's hitBVH (P5/fsh:254-306) walks a binary tree of 48-byte nodes with three dependent fetches
// per step.  The accel policy only has to find the globally closest accepted triangle (capi.cu decides by the
// deferral rule whether that is also the shader's answer), so its tree is free in shape, order and box
// precision as long as every child box is a SUPERSET of the exact (2*delta-inflated) box of its sub-tree:
//
//   record = 20 words = 80 bytes, 16-byte aligned, read with five 128-bit loads
//     w0..2   origin.xyz (float)      one quantisation step below the lowest child plane of the node
//     w3      ex | ey << 8 | ez << 16 | imask << 24
//             ex, ey, ez              biased IEEE exponents of the per-axis scale: scale_a = as_float(e_a << 23), a power
//                                     of two in [2^-126, 2^127], >= W8 minimum step of the scene (fp error bound below)
//             imask                   bit s: slot s holds an inner child
//     w4      child_base              node index of the first inner child; inner children are numbered consecutively
//                                     in slot order: child of slot s = child_base + popc(imask & ((1 << s) - 1))
//     w5      tri_base                first triangle (accel order) of the node's leaf children, consecutive in slot order
//     w6..11  qlo_x[8] qlo_y[8] qlo_z[8]   low planes of the eight slots, one byte each (slot s = byte s)
//     w12,13  meta[8]                 leaf slot: (count << 5) | offset of its first triangle from tri_base (count 1..4,
//                                     offset 0..28); inner or empty slot: 0
//     w14..19 qhi_x[8] qhi_y[8] qhi_z[8]   high planes
//   plane value = origin + q * scale; an empty slot has qlo = 255, qhi = 0 (inverted, never hit).
//
// Decode (one FMA per plane, same formula on host model and device):
//     B = as_float(e << 23) * inv_d   (= scale * inv_d, exact: scale is a power of two)
//     A = fma(-2^15, B, (origin - o) * inv_d)
//     f = as_float(0x47000000 | q << 8) = 2^15 + q        (one PRMT on the device: the byte goes to mantissa bits 8..15)
//     t = fma(f, B, A)             = (origin + q*scale - o) * inv_d up to rounding (the 2^15 * B terms cancel exactly)
// Conservativeness: the builder stores floor(x - W8_SLACK_STEPS) for low planes and ceil(x + W8_SLACK_STEPS) for high
// planes (x = exact plane in steps).  Rounding error of the decode: A is rounded once at magnitude <= 2^15 * B + |t|, i.e.
// 2^-9 step + 2^-24 |t|; (origin - o) * inv_d carries 2 * 2^-24 * |origin - o| * |inv_d|; the final FMA 2^-24 |t|.  The
// builder keeps scale >= W8_MIN_STEP_REL * max|coordinate| and the kernel only traces rays with
// |o| <= W8_ORIGIN_LIMIT_REL * max|coordinate| and 2^-60 <= |inv_d| <= the scene's decode range on this tree (all others go to
// the exact kernel), so with |plane|, |o| <= 5 max|coordinate| the total stays below 4 * 2^-24 * 5 * max|coordinate| * |inv_d|
// + 2^-9 step < 0.16 step + 0.002 step < W8_SLACK_STEPS (0.25).
// Decode range: the bound above holds only while every term is finite.  2^15 * B = 2^15 * scale * |inv_d| reaches 2^128 for
// large scenes (a root scale of 2^19, a scene 10^8 wide, overflows at |inv_d| = 2^94): A becomes +-inf, every slot's exit
// distance -inf, and the ray misses the whole tree.  ezrt_quant_inv_limit (accel_w8.cpp) therefore derives the limit on
// |inv_d| per scene from the largest per-axis scale of the tree and max|coordinate|: a power of two, at most W8_INV_LIMIT, that
// keeps 2^15 * scale * |inv_d| and 5 * max|coordinate| * |inv_d| at or below 2^124 (the Q16 nodes: 2^23 * scale).
//
// Slot order ("octant order", after Ylitie, Karras, Laine 2017): the builder places a child in the slot whose
// corner direction (bit a of the slot index set = towards +axis_a) matches the child's offset from the node
// centre best; a ray visits hit slots in descending (slot ^ near_mask), near_mask bit a = 1 iff d_a >= 0, so
// children on the side the ray comes from go first, without sorting distances.  The bit significance of the
// axes (which axis decides first) is a per-scene permutation: the axis of largest scene extent is bit 2.
#ifndef EZRT_W8_NODE_H
#define EZRT_W8_NODE_H

#include <stdint.h>

#define W8_NODE_WORDS 20
#define W8_NODE_BYTES 80
#define W8_MAX_LEAF_TRIS 4            // triangles per leaf slot (meta count field)
#define W8_MAX_NODE_TRIS 32           // triangles of all leaf slots of one node (bits of the triangle mask)
#define W8_SLACK_STEPS 0.25                  // outward slack of the stored planes, in quantisation steps
#define W8_DECODE_BIAS 32768.0f              // 2^15: f = as_float(W8_DECODE_BITS | q << 8) = 2^15 + q
#define W8_DECODE_BITS 0x47000000u
#define W8_MIN_STEP_REL 7.62939453125e-06f   // 2^-17: smallest quantisation step relative to max |coordinate|
#define W8_ORIGIN_LIMIT_REL 4.0f
#define W8_INV_LIMIT 7.9228162514264338e28f  // 2^96: the largest decode range of any scene (SceneDev::quant_inv_limit)
#define W8_INV_MIN 8.6736173798840355e-19f   // 2^-60: ... or a smaller one (no underflow)

#define W8_LOCAL_STACK 48                    // stack entries beyond the shared-memory part (local memory)

#define W8_W_ORIGIN 0
#define W8_W_EXP_IMASK 3
#define W8_W_CHILD_BASE 4
#define W8_W_TRI_BASE 5
#define W8_W_QLO 6
#define W8_W_META 12
#define W8_W_QHI 14

// bits of the scale of axis a (0..2) from word W8_W_EXP_IMASK: the exponent byte moved to the float's exponent field
#define W8_SCALE_BITS(w, a) ((((uint32_t)(w) >> (8 * (a))) & 0xffu) << 23)

#endif
