// match_tc.cuh — interface between the tensor-core nomination pass (match_tc.cu)
// and the exact decision logic (match.cu).
#pragma once
#include "common.cuh"
#include <vector>

struct TcImage {
  long long row0;   // first descriptor row of this image in the featureset buffer
  int n;            // real rows
  int n_pad;        // rows padded to a multiple of 256
  int blk0;         // first 128-row block of this image in the operand buffers
};

struct TcTop2 { float m1, m2; int idx; int pad; };   // approximate best / second-best d^2 and argmin

#define TC_CAND_CAP 16     // candidate columns kept per gathered row (more -> full exact re-scan)

struct TcTask {       // one CTA: 128 query rows against every target row
  int q_blk;          // operand block holding the query rows
  int q_row0, q_n;    // top2: first query row of this block within its image, rows in the image
                      // filter: index of the block's first gathered row, real rows in the block
  int t_blk0, t_blocks;  // target image: first block, number of blocks (even)
  int t_n, t_pad;     // real target rows; filter: first list slot of this block; first pass: the first
                      // target column of this task (a task may cover only a range of the target tiles)
  long long res_off;  // top2: where the query image's results start; filter: side index
};

struct TcGatherSide {  // per query side, for the gathered second pass
  long long q_base;    // descriptor row of the side's first query (norms index)
  long long res_off;   // approx / RowInfo offset of the side
  long long list_off;  // first slot of the side's request list
  int q_blk0;          // operand block of the side's first query row
  int t_blk0, t_blocks, t_n;
};

struct TcFilter {       // device buffers of one gathered pass
  unsigned char* gq;    // gathered query blocks
  TcTask* tasks;        // built on the device
  int* n_tasks;         // device counter
  const TcGatherSide* gsides;
  const int* list_rows;
  const TcTop2* approx;
  int2* g_meta;         // (side, row) per gathered row, (-1,-1) for padding
  int* g_thr;
  int* cand_cnt;
  int* cand;            // [gathered rows][TC_CAND_CAP]
};

struct TcOperands {
  DevBuf<TcImage> d_imgs;
  DevBuf<float> d_norms;           // |x|^2 per descriptor row (f32)
  DevBuf<unsigned> d_maxnorm;      // bits of max |x|^2
  DevBuf<unsigned char> qbuf;      // query-form fp16 blocks
  DevBuf<unsigned char> tbuf;      // target-form fp16 blocks
};

int  tc_prepare(pano_ctx* ctx, const float* d_desc, const std::vector<TcImage>& imgs, TcOperands* ops);
int  tc_run_top2(pano_ctx* ctx, const TcOperands* ops, const TcTask* d_tasks, int n_tasks, TcTop2* d_res);
int  tc_run_filter(pano_ctx* ctx, const TcOperands* ops, const TcFilter* f, int max_blocks);
int  tc_run_nominate(pano_ctx* ctx, const TcOperands* ops, const TcFilter* f, int max_blocks, TcTop2* d_res);
size_t tc_block_bytes();
