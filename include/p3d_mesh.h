/*
 * p3d_mesh.h - C ABI of the marching-cubes mesh extraction (SURVEY.md 8f-2 -> 8f-4: the geometry stage of the eval).
 *
 * The reference meshes the 256^3 density volume on the host: `marching_cubes` (_util/eg3d_metrics3d.py:186-211) copies
 * the densities and the whole 32-channel colour volume to the host, runs skimage's Lewiner marching cubes and looks up
 * each vertex colour in a Python loop.  Here the mesh is extracted on the device in two passes with a device-wide
 * exclusive scan between them; DESIGN.md section 2 ("Marching cubes") states the rules (vertex order, face rule with
 * the asymptotic decider, winding, degenerate removal) that the kernels and the CPU oracle (oracle/mesh_oracle.py) share.
 *
 * The volume is a dense C-contiguous fp32 (d0, d1, d2) array, every side >= 2, at most 2^30 nodes.  Positions are in index
 * space (a, b, c).  Device pointers; return codes / p3d_last_error() as in p3d_render.h.
 */
#ifndef P3D_MESH_H_
#define P3D_MESH_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Scratch that must stay untouched between p3d_mc_count and p3d_mc_emit for a (d0, d1, d2) volume (bytes); 0 on error. */
size_t p3d_mc_workspace_bytes(int64_t d0, int64_t d1, int64_t d2);

/* Pass 1: per node its sign-change edges, per cell its non-degenerate triangles, then the exclusive scan of both.
   counts2 (device, 2 x int64) receives (vertex count V, triangle count F); read it before allocating the outputs. */
int p3d_mc_count(const float* vol, int64_t d0, int64_t d1, int64_t d2, float level, void* workspace, size_t workspace_bytes,
                 int64_t* counts2, void* stream);

/* Pass 2 (same volume, level and workspace as the p3d_mc_count call): writes
     verts (V,3) fp32 index-space positions;  faces (F,3) int32, right-hand normal pointing from inside to outside;
     normals (V,3) fp32 or NULL;  values (V) fp32 or NULL;  floor_node (V) int64 flat index of floor(position) or NULL.
   Writes nothing when V or F is 2^31 or more (faces are int32). */
int p3d_mc_emit(const float* vol, int64_t d0, int64_t d1, int64_t d2, float level, const void* workspace,
                size_t workspace_bytes, float* verts, int32_t* faces, float* normals, float* values, int64_t* floor_node,
                void* stream);

/* Lattice coordinates of volume elements for the colour lookup: element f = (a*R + b)*R + c of the flipped volume that
   p3d_volume_query returns is the reference's create_samples point n = ((R-1-a)*R + b)*R + c (eg3d_metrics3d.py:70-92),
   reproduced bit for bit.  flat (n_points) int64 -> coords (n_points, 3) fp32, ready for p3d_decode_points. */
int p3d_mc_lattice_coords(const int64_t* flat, int64_t n_points, int32_t resolution, double cube_length, float* coords,
                          void* stream);

#ifdef __cplusplus
}
#endif
#endif /* P3D_MESH_H_ */
