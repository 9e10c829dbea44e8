/* n2m_b200_texture.h -- C ABI of the stage-1 texture export of libn2m_b200.so (csrc/texture.cu; host side nerf2mesh_b200/texture.py).
 *
 * The reference's NeRFRenderer.export_stage1 (nerf/renderer.py:298-468) bakes the appearance features of the final mesh into a UV atlas:
 * rasterize the mesh in UV space at (h, w) = ssaa * (h0, w0), interpolate the positions, evaluate `geo_feat` = sigmoid(color_net(...)),
 * 6 channels, on the covered texels, quantise to uint8, inpaint a 32-texel gutter from the nearest boundary texels, down-sample.
 * The UV raster is n2m_rasterize with clip positions (vt * 2 - 1, 0, 1) and triangles ft; the hash-grid gather is n2m_s0_encode_points.
 *
 *   n2m_s1_bake_points   covered texels of rows [y0, y1) of the UV raster `rast` [H,W,4] (rast[...,3] > 0) -> pix [cap] (texel index
 *       y * W + x) and pts [cap,3] = dr.interpolate(verts, rast, tri) at those texels (tri = the POSITION triangles f, indexed by the
 *       triangle id ft rasterized; the fp32 expression of n2m_interpolate_forward, bit-identical), contracted (renderer.py:25-32) when
 *       `contract` != 0.  counters (>= 4 int32, reset here): [0] covered texels of the band, [1] min([0], cap) -- the point count
 *       n2m_s0_encode_points reads --, [2] overflow flag.  The order of the points within a band is not deterministic; the image is.
 *   n2m_s1_geo_feat      color_net on tensor cores over the n2m_s0_encode_points tiles enc_tiles [Pcap/128 tiles] of points
 *       [0, counters[1]): the colour rounds of n2m_s0_mlp_fwd (same GEMM shapes, K order and fp16 rounding points), sigmoid, then
 *       feats[pix[k] * 6 + c] = (uint8_t)(f_c * 255) (truncation, as numpy's astype).  feats_f32 [Pcap,6] (nullable) receives the
 *       features before quantisation.
 *   n2m_s1_inpaint       in place on feats [H*W,6] uint8 with the coverage mask [H*W] (0 / 1), renderer.py:378-394 without a KD-tree:
 *       search  = mask texels within L1 distance 3 of a non-mask texel or of the image border (mask & ~binary_erosion(mask, 3));
 *       inpaint = non-mask texels within L1 distance 32 of a mask texel (binary_dilation(mask, 32) & ~mask);
 *       every inpaint texel copies the 6 bytes of its Euclidean-nearest search texel; ties go to the smallest source row, then the
 *       smallest source column.  Texels that are neither mask nor inpaint are set to 0; mask texels are left as they are.
 *       scratch: 3 * H * W bytes.  source [H*W] (nullable) receives the source texel of every inpaint texel and -1 elsewhere.
 *   n2m_s1_ssaa_down2    feats [h0*ssaa, w0*ssaa, 6] -> feat0 = channels 0-2, feat1 = channels 3-5, each [h0,w0,3] uint8; ssaa 2: the
 *       mean of each 2x2 block, (a + b + c + d + 2) >> 2 (cv2.resize INTER_LINEAR at exactly half size); ssaa 1: a copy.
 *
 * Rendering the exported asset as the viewer does (the fragment shader of renderer.html:54-160, every cascade in one depth buffer):
 *   n2m_s1_asset_shade   one thread per sample of rast [num_pixels,4] (n2m_rasterize of all cascades concatenated: verts [V,3] world space,
 *       tri [F,3], face f of cascade c for face_offsets[c] <= f < face_offsets[c+1], face_offsets [cascades+1] on the device).  A covered
 *       sample interpolates the OBJ texture coordinate (s, t) = st [Nt,2] at ft [F,3] (t = the file's 1 - v) with rast's barycentrics,
 *       u s0 + v s1 + (1 - u - v) s2 with every product and sum rounded separately, and fetches the nearest texel of cascade c's RGB
 *       uint8 textures feat0[c] / feat1[c] [H_c,W_c,3] (device arrays of device pointers; tex_size [cascades,2] = (H_c, W_c) on the
 *       device) as three.js NearestFilter + flipY + clamp-to-edge does: column clamp(floor(s W_c)), row clamp(H_c - 1 - floor(t H_c)),
 *       value / 255.  mode 1 ('diffuse'): the feat0 colour; otherwise specular_net in fp32 on [normalize(x - cam), feat1]: mlp = the
 *       weights [32,6] then [3,32] ([out, in], 288 floats on the device), ReLU, sigmoid; mode 2 ('specular'): that output, mode 3 ('full'):
 *       clamp(diffuse + specular, 0, 1).  img [num_pixels] float4 = (r, g, b, 1) at covered samples, 0 elsewhere -- the input of
 *       n2m_antialias_forward (C = 4) and n2m_s1_render_compose (include/n2m_b200_raster.h).
 */
#ifndef N2M_B200_TEXTURE_H
#define N2M_B200_TEXTURE_H

#include "n2m_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

int n2m_s1_bake_points(const float* rast, const float* verts, const int32_t* tri, uint32_t W, uint32_t y0, uint32_t y1, uint32_t cap,
                       uint32_t contract, int32_t* counters, int32_t* pix, float* pts, n2m_stream_t stream);
int n2m_s1_geo_feat(const void* enc_tiles, const int32_t* counters, uint32_t Pcap, const void* wpack, const int32_t* pix, uint8_t* feats,
                    float* feats_f32, n2m_stream_t stream);
int n2m_s1_inpaint(uint8_t* feats, const uint8_t* mask, uint32_t H, uint32_t W, uint8_t* scratch, int32_t* source, n2m_stream_t stream);
int n2m_s1_ssaa_down2(const uint8_t* feats, uint32_t h0, uint32_t w0, uint32_t ssaa, uint8_t* feat0, uint8_t* feat1, n2m_stream_t stream);
int n2m_s1_asset_shade(const float* rast, uint32_t num_pixels, const float* verts, const int32_t* tri, const float* st, const int32_t* ft,
                       const int32_t* face_offsets, uint32_t cascades, const void* const* feat0, const void* const* feat1, const int32_t* tex_size,
                       const float* mlp, float cam_x, float cam_y, float cam_z, uint32_t mode, float* img, n2m_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* N2M_B200_TEXTURE_H */
