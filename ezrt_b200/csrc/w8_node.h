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
// Bundle bound (the camera pass, extend_w8_bundle in device_functions.cuh; the same arithmetic in tools/w8_model.cpp): one
// interval test per slot decides for all member rays r of a (sub-)bundle at once whether one of them may reach the slot.
//     per member ray: the float o_r, v_r = EZ_DIV(1, d_r) the per-ray decode uses (finite and non-zero: the load gate)
//     per axis a: [omin, omax] of o_a,r and [vmin, vmax] of v_a,r over the members; the axis constrains the test only when all
//                 members have d_a >= 0 ("pos") or all have d_a < 0 (sub-bundles always do: their v_a,r share one sign)
//     planes, widened by W8_SLACK_STEPS and rounded outward: lo = rd(origin + (q_lo - 0.25) scale), hi = ru(origin + (q_hi + 0.25) scale)
//                 ((q -+ 0.25) scale is exact: q has 8 bits, scale is a power of two)
//     near plane pn = pos ? lo : hi, far plane pf = pos ? hi : lo
//     xe = pos ? rd(pn - omax) : ru(pn - omin)          entry = rd(xe * (xe >= 0 ? vmin : vmax))
//     xx = pos ? ru(pf - omin) : rd(pf - omax)          exit  = ru(xx * (xx >= 0 ? vmax : vmin))
//     hit iff max(entry_x, entry_y, entry_z, 0) <= min(exit_x, exit_y, exit_z, L),   L = max over members of the per-ray limit
// (rd / ru: round toward -inf / +inf).  For every member, (pn - o_a,r) v_a,r >= entry and (pf - o_a,r) v_a,r <= exit: the
// product is monotonic in each factor on the box [omin, omax] x [vmin, vmax], and the chosen corner is its minimum (maximum),
// with every rounding outward.  The per-ray decode of the same planes differs from (plane - o) v by less than 0.162 step
// (above), less than the 0.25 step the bundle widens each plane by.  So a slot the per-ray test of any member hits, at any
// limit <= L, is hit by the bundle test.  The bound is only as tight as [vmin, vmax]: where a component of d crosses zero
// its 1/d spreads without bound, which is why a sub-bundle keeps each component of 1/d within a factor 2 of its leader's.
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
// The tree the collapse starts from and what it weighs (accel_w8.cpp, capi.cu): the binary SAH tree is built down to
// W8_BINARY_LEAF_TRIS triangles per leaf, so that the collapse, not the binary builder, decides every leaf slot (Ylitie et al.
// 2017); a triangle test is priced at W8_COST_TRI node visits.  Measured on an H100 (700 W), a test costs 1.16 visits in the
// bounce kernel; on single-triangle leaves, prices from 0.4 to 1.6 predict bounce-kernel cycles within 1.5 % of each other
// (tools/w8_model.cpp sweep), and 0.4 keeps the larger leaf slots that load the cooperative triangle step.  DESIGN.md section 6.
#define W8_BINARY_LEAF_TRIS 1
#define W8_COST_TRI 0.4
#define W8_SLACK_STEPS 0.25                  // outward slack of the stored planes, in quantisation steps
#define W8_DECODE_BIAS 32768.0f              // 2^15: f = as_float(W8_DECODE_BITS | q << 8) = 2^15 + q
#define W8_DECODE_BITS 0x47000000u
#define W8_MIN_STEP_REL 7.62939453125e-06f   // 2^-17: smallest quantisation step relative to max |coordinate|
#define W8_ORIGIN_LIMIT_REL 4.0f
#define W8_INV_LIMIT 7.9228162514264338e28f  // 2^96: the largest decode range of any scene (SceneDev::quant_inv_limit)
#define W8_INV_MIN 8.6736173798840355e-19f   // 2^-60: ... or a smaller one (no underflow)

#define W8_LOCAL_STACK 48                    // stack entries beyond the shared-memory part (local memory)
#define W8_BUNDLE_STACK 64                   // entries of a warp's stack in the camera pass (shared memory): a lane's 16 + 48

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
