// bwt_msd.h -- constants and entry point of the MSD + shared-memory bucket sort path of the forward BWT (bwt_msd.cu).
#pragma once
#include "ctx.h"

#define MSD_TILE 4096      // text bytes per scatter tile
#define MSD_THREADS 256
#define MSD_ITEMS 16
#define MSD_CTAS_PER_SM 5
#define MB_THREADS 1024    // one persistent CTA per SM
#define MB_ITEMS 10
#define MB_BUF (MB_THREADS * MB_ITEMS)  // records per shared-memory buffer (80 KiB); two buffers: sort one, prefetch the next
#define MB_CAP (MB_BUF - 2)             // largest (block, first byte) bucket the path takes
#define MB_CELL_BITS 14
#define MB_CELLS (1u << MB_CELL_BITS)   // interpolation cells per bucket
#define MB_MAXCELL 512u                 // a fuller cell means the keys are far from uniform: give up, the LSD path takes the batch

struct MsdBlk {
  u32 a, a2;  // symbols in use in the block, squared
  u64 S;      // floor(2^64 / a^4): scaled key = (key * S) >> 32
};

// d_ctl: u32[4] zeroed by the caller: [0] = members of tie groups written to the tie list, [1] = a cell exceeds MB_MAXCELL,
// [2] = a bucket exceeds MB_CAP (nothing was done), [3] = non-empty buckets (length of the work list).
void bwt_msd_launch(Ctx& c, const u8* d_T, u8* d_U, const u32* d_n, u32 nblk, u32 n_max, u64 n_total, const u32* d_hist, u64* d_rec,
                    u32* d_pidx, u32* d_tie_head, u32* d_tie_idx, u32* d_ctl);
