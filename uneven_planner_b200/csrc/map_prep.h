// map_prep.h -- cloud preprocessing shared by the host and the CUDA UnevenMap builders (internal to libualm).
#pragma once

#include <cstdint>
#include <vector>

#include "map_cell.h"

// CropBox + 1 cm VoxelGrid (uneven_map.cpp:133-143) + uniform XY bin grid (bin = largest ellipsoid semi-axis) of the cloud
struct UalmMapHostPrep {
    std::vector<float> pts;   // bin-sorted, xyz interleaved
    std::vector<int> start;   // nx*ny+1
    int nx = 1, ny = 1;
    double x0 = 0, y0 = 0, inv = 1, box_r = 1;
    UalmMapPrep view(double ex, double ey, double ez, int iter_num) const
    {
        UalmMapPrep g;
        g.pts = pts.data(); g.start = start.data(); g.npts = (int)(pts.size() / 3); g.nx = nx; g.ny = ny;
        g.x0 = x0; g.y0 = y0; g.inv = inv; g.box_r = box_r;
        g.einv[0] = 1.0 / ex; g.einv[1] = 1.0 / ey; g.einv[2] = 1.0 / ez;
        g.iter_num = iter_num;
        return g;
    }
};
// (cx, cy): the centre of the grid the cloud is for; the crop box is [cx - 10, cx + 10] x [cy - 10, cy + 10] x [-0.01, 5]
void ualm_map_preprocess(const float *pin, int64_t npts, double ex, double ey, double ez, double cx, double cy, UalmMapHostPrep &out);
// centre of grid g along axis k (0 = x, 1 = y); exactly 0 for every grid ualm_map_geometry makes
inline double ualm_map_centre(const ualm_map_geom_t &g, int k) { return (g.origin[k] + g.max_boundary[k]) / 2.0; }
