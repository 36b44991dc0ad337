// b200q_decode_plan.h — decode launches (b200q_decode.cu): every mat-vec launch is planned on the host before anything is launched.
// Used by the decode launchers (b200q_decode.cu, b200q_wire.cu), by the C ABI (b200q_api.cu) and, for the shared-memory opt-in, by the GEMMs.
// A plan names the kernel, its template arguments and its launch shape.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>
#include "b200q_internal.h"

// the activations of the decode mat-vecs quantised in shared memory: [ncols K int8][ncols K/32 f32 d][ncols K/32 i32 sums]
static inline size_t b200q_mmvq_x_bytes(int64_t ncols, int64_t K) { return (size_t)ncols * K + (size_t)ncols * (K / 32) * 8; }
// the most columns of length K whose image one mat-vec launch holds (~200 KB of the 227 KB a CTA may use)
static inline int64_t b200q_mmvq_max_cols(int64_t K) {
    const size_t col = b200q_mmvq_x_bytes(1, K);
    return col ? (int64_t)((200 * 1024) / col) : INT32_MAX;
}

// ring geometry of a type (k_mmvq_ring)
struct ring_geom {
    int n_planes;                 // block planes staged through the ring (the per-row scale plane is read directly)
    int b8[4];                    // bytes per 8 items (256 weights) of plane p
    int seg_off[4];               // byte offset of plane p inside a stage
    int stage_bytes;              // 16-byte aligned
    int n_stages;                 // S
    int row_plane;                // index of the per-row plane in b200q_planes::p, or -1
    int merged;                   // 1: the row is ONE segment, so the two rows of a pair are adjacent inside every plane and travel as one bulk copy per
                                  //    plane (half as many copies in flight: tools/membench.cu `r` shows the bandwidth falling with the copy count);
                                  //    the stage is then laid out plane-major [p0 row0 | p0 row1 | p1 row0 | p1 row1 ...]
    int row1[4];                  // byte offset of row 1 of the pair relative to row 0, per plane
};

// one decode launch: the kernel, its template arguments and its launch shape
enum { B200Q_MMVQ_LDG = 0, B200Q_MMVQ_RING = 1, B200Q_MMVQ_WIRE = 2 };
struct b200q_mmvq_plan {
    int kernel;                                       // B200Q_MMVQ_*: k_mmvq / k_mmvq_id, k_mmvq_ring, k_wire_mmvq / k_wire_mmvq_id
    int ncols; bool upgate, multi, pair, tp; int q8;  // template arguments (k_mmvq_ring<T, ncols, upgate, multi, pair, tp, q8>)
    ring_geom g; int ncw;                             // ring: geometry (g.n_stages = stages), consumer warps
    dim3 grid, block; size_t smem;                    // dynamic shared memory
    int tp_rowbuf_off, tp_rowbuf_rows;                // ring, tp.out: the CTA's row buffer (mmvq_args)
};
// Dense decode: plans d (plan_mmvq), then launches it; `plan`: what was launched.  A q8 hand-off the shape is not eligible for is
// planned as the plain launch (q8 = 0).
int b200q_launch_mmvq(const b200q_mmvq_desc & d, cudaStream_t st, b200q_mmvq_plan * plan = nullptr);
int b200q_launch_wire_mmvq(const b200q_mmvq_desc & d, const b200q_mmvq_plan & p, cudaStream_t st);
// the launch shape of k_mmvq_id / k_wire_mmvq_id: 0, or -2 when the activation columns do not fit shared memory
int b200q_plan_mmvq_id(const b200q_mmvq_id_desc & d, b200q_mmvq_plan & p);
int b200q_wire_check(int type, int64_t M, int64_t K);

// raise a kernel's dynamic shared-memory limit on the current device to `bytes` (never lowers it; nothing to do up to 48 KB): false on failure
bool b200q_opt_in_smem(const void * kernel, size_t bytes);
// launch of a decode kernel with its one argument struct `arg`, as a programmatic dependent launch when `pdl`
int b200q_launch_pdl(const void * kernel, dim3 grid, dim3 block, size_t smem, void * arg, bool pdl, cudaStream_t st);
