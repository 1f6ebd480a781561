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
