// blend_rows.cuh — the parts of blend.cu's row-strip blend streams that the strip sweep (blend_sweep.cu) drives.
#pragma once
#include <vector>

#include "common.cuh"

// Summed half-widths H of the multiband level blurs (the strip halo, pano_blend_rows_dev), or -kw for a window
// wider than the tap table.  0 for bands < 2.
int blend_halo(int bands, const pano_params* p);
// The one rule for whether rows [row0, row1) of an oh-row canvas read image `im` (pano_blend_stream_needs,
// pano_blend_rows_rgb8_dev): the whole canvas reads every image; multiband, the ROI clipped to
// [row0 - H, row1 + H) keeps a row; linear, the ROI's rows [y0, y1] meet the strip.
bool blend_strip_reads(const pano_blend_image& im, int bands, int halo, int oh, int row0, int row1);
// pano_blend_stream_create_rows with the device projection tables `shared_tab` (blend_sweep_tables' values,
// or null to build them for this stream).
int blend_stream_open(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                      const pano_params* p, int ow, int oh, int row0, int row1, const double* shared_tab,
                      pano_blend_stream** out);
// Validates a blend of the whole canvas as pano_blend_stream_create does and returns its host projection
// tables (empty for the flat projection).
int blend_sweep_tables(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                       const pano_params* p, int ow, int oh, std::vector<double>* tab);
// Cylinder mode's perspective correction of output rows [row0, row1) of a w×h canvas (cylstitcher.cc:139-180, with
// inv its `inv`) into d_out (from row0 on), the mosaic's rows [b0, b0 + band rows) in d_band.  The band must hold
// every row persp_band gives for these rows.
int persp_correct_rows(pano_ctx* ctx, const float* d_band, int b0, const double inv[9], int w, int h,
                       const pano_params* p, float* d_out, int row0, int row1);
// The cylinder warps of a cylinder stream's sources (pano_blend_stream_create_cyl): each source's shape, its
// inverse map and the offset of its column tables in `tabs` (col_x then col_cos, 16 B per warped column).
struct CylTabs {
  std::vector<CylMap> maps;
  std::vector<size_t> off;
  std::vector<int> w, h;
  std::vector<double> tabs;
};
// Validates the sources as pano_blend_stream_create_cyl does (every warp must have imgs[k]'s shape) and builds
// their tables.
int cyl_tabs(pano_ctx* ctx, int n, const pano_blend_image* imgs, const int* src_w, const int* src_h, double h_factor,
             const pano_params* p, CylTabs* ct);
// blend_stream_open for rows [row0, row1) of a cylinder stream over ct's sources.  d_cyl_tab: ct.tabs on the
// device, shared by many streams, or null to upload them for this stream.
int blend_stream_open_cyl(pano_ctx* ctx, int n, const pano_blend_image* imgs, const pano_blend_geom* g, int bands,
                          const pano_params* p, int ow, int oh, int row0, int row1, const double* shared_tab,
                          const CylTabs& ct, const double* d_cyl_tab, pano_blend_stream** out);
