// m3t_b200_render.cu — k_render: one CTA per focused renderer. Focus (FocusedRenderer::CalculateProjectionMatrix,
// renderer.cpp:348-405), rasterisation of every geometry body into a shared-memory z-buffer, write-out of the focused
// depth / silhouette images and of the renderer-image records k_track / k_histogram read. Float32 throughout, one
// rounding per operation in the order written (the library is built with -fmad=false); DESIGN.md §3 "k_render" states
// the contract and tests/render_reference.py restates it.
#include <cfloat>

#include "m3t_b200_raster.cuh"
#include "m3t_b200_render.cuh"

namespace m3tb {

__global__ void __launch_bounds__(kRenderThreads) k_render(const __grid_constant__ RenderArgs a) {
  extern __shared__ uint32_t zbuf[];
  __shared__ float sP[6];   // P00, P02, P11, P12, P22, P23 (renderer.cpp:397-404)
  __shared__ float sM[16];  // P * world2camera * geometry2world, row-major
  __shared__ int s_any;
  const int r = a.render_list[blockIdx.x];
  const RendererDev& R = a.renderers[r];
  const int S = R.image_size, n_pix = S * S;
  const CameraDev& cam = R.camera_kind == 0 ? a.color_cams[R.camera] : a.depth_cams[R.camera];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n_warps = blockDim.x >> 5;
  for (int p = tid; p < n_pix; p += blockDim.x) zbuf[p] = 0xFFFFFFFFu;  // glClear: depth 1.0, no body

  // ---- focus: FocusedRenderer::CalculateProjectionMatrix (renderer.cpp:348-405) -------------------------------------
  if (tid == 0) {
    const float* w = cam.w2c;
    float u_min = FLT_MAX, u_max = FLT_MIN, v_min = FLT_MAX, v_max = FLT_MIN;  // numeric_limits<float>::min() as written
    int any = 0;
    for (int k = 0; k < R.n_referenced; ++k) {
      const int b = a.referenced_bodies[R.first_referenced + k];
      int vis = 0;
      const float rr = a.geometry[b].radius;
      const float* p = a.poses + 12 * b;
      const float x = w[0] * p[3] + w[1] * p[7] + w[2] * p[11] + w[3];
      const float y = w[4] * p[3] + w[5] * p[7] + w[6] * p[11] + w[7];
      const float z = w[8] * p[3] + w[9] * p[7] + w[10] * p[11] + w[11];
      if (!(z < rr * 1.5f || z - rr < R.z_min || z + rr > R.z_max)) {
        const float abs_x = fabsf(x), abs_y = fabsf(y);
        const float x2 = x * x, y2 = y * y, z2 = z * z, r2 = rr * rr, rz = rr * z;
        const float z2_r2 = z2 - r2;
        const float z3_zr2 = z2_r2 * z;
        const float r_u = cam.fu * (abs_x * r2 + rz * sqrtf(z2_r2 + x2)) / z3_zr2;
        const float r_v = cam.fv * (abs_y * r2 + rz * sqrtf(z2_r2 + y2)) / z3_zr2;
        const float center_u = x * cam.fu / z + cam.ppu;
        const float center_v = y * cam.fv / z + cam.ppv;
        const float u_min_body = center_u - r_u, u_max_body = center_u + r_u;
        const float v_min_body = center_v - r_v, v_max_body = center_v + r_v;
        if (!(u_min_body > float(cam.width) || u_max_body < 0.0f || v_min_body > float(cam.height) || v_max_body < 0.0f)) {
          u_min = u_min_body < u_min ? u_min_body : u_min;  // std::min(a, b) = b < a ? b : a
          u_max = u_max < u_max_body ? u_max_body : u_max;  // std::max(a, b) = a < b ? b : a
          v_min = v_min_body < v_min ? v_min_body : v_min;
          v_max = v_max < v_max_body ? v_max_body : v_max;
          vis = 1;
          any = 1;
        }
      }
      a.visible[R.first_referenced + k] = vis;
    }
    const float du = u_max - u_min, dv = v_max - v_min;
    const float d = (du < dv ? dv : du) * 1.05f;  // kImageSizeSafetyMargin
    RenderOutDev o;
    o.corner_u = 0.5f * (u_min + u_max - d);
    o.corner_v = 0.5f * (v_min + v_max - d);
    o.scale = float(S) / d;
    o.projection_term_a = R.z_max * R.z_min * 65535.0f / (R.z_max - R.z_min);  // renderer.cpp:567-570
    o.projection_term_b = R.z_max * 65535.0f / (R.z_max - R.z_min);
    a.out[r] = o;
    const float ppu_scaled = (cam.ppu - o.corner_u) * o.scale;
    const float ppv_scaled = (cam.ppv - o.corner_v) * o.scale;
    sP[0] = 2.0f * cam.fu / d;
    sP[1] = 2.0f * (ppu_scaled + 0.5f) / float(S) - 1.0f;
    sP[2] = 2.0f * cam.fv / d;
    sP[3] = 2.0f * (ppv_scaled + 0.5f) / float(S) - 1.0f;
    sP[4] = (R.z_max + R.z_min) / (R.z_max - R.z_min);
    sP[5] = -2.0f * R.z_max * R.z_min / (R.z_max - R.z_min);
    s_any = any;  // no visible body: the matrix is not finite, nothing is drawn, the images stay cleared
  }
  __syncthreads();

  // ---- raster: every geometry body in draw order, triangles over the warps ------------------------------------------
  if (s_any) {
    const float half = 0.5f * float(S);
    for (int g = 0; g < R.n_geometry; ++g) {
      const int b = a.geometry_bodies[R.first_geometry + g];
      const GeometryDev& G = a.geometry[b];
      if (tid == 0) {
        float g2w[12], T[12];
        PoseMul(a.poses + 12 * b, G.geometry2body, g2w);  // Body::geometry2world_pose (body.cpp:88)
        PoseMul(cam.w2c, g2w, T);                         // world2camera * geometry2world
        // P * [T; 0 0 0 1]; the products with P's zero entries are left out (adding an exact zero changes no sum)
        for (int c = 0; c < 4; ++c) {
          sM[c] = sP[0] * T[c] + sP[1] * T[8 + c];
          sM[4 + c] = sP[2] * T[4 + c] + sP[3] * T[8 + c];
          sM[8 + c] = sP[4] * T[8 + c];
          sM[12 + c] = T[8 + c];
        }
        sM[11] = sM[11] + sP[5];
      }
      __syncthreads();
      float M[16];
#pragma unroll
      for (int k = 0; k < 16; ++k) M[k] = sM[k];
      const unsigned draw_index = unsigned(g);
      auto frag = [&](int i, int j, unsigned d16) { atomicMin(zbuf + j * S + i, (d16 << 16) | draw_index); };
      for (int t = warp; t < G.n_triangles; t += n_warps)
        DrawTriangle(M, G.triangles + 9 * t, G.enable_culling, S, S, half, half, frag, lane);
      __syncthreads();  // sM is rewritten for the next body
    }
  }
  __syncthreads();

  // ---- write-out ---------------------------------------------------------------------------------------------------
  for (int p = tid; p < n_pix; p += blockDim.x) {
    const int i = p % S, j = p / S;
    const uint32_t v = zbuf[p];
    const unsigned d16 = v >> 16;
    int id = 0;
    if (d16 != 0xFFFFu) {
      const GeometryDev& G = a.geometry[a.geometry_bodies[R.first_geometry + int(v & 0xFFFFu)]];
      id = R.id_type == RID_REGION ? G.region_id : G.body_id;
    }
    reinterpret_cast<uint16_t*>(reinterpret_cast<uint8_t*>(R.depth) + size_t(j) * R.depth_pitch)[i] = uint16_t(d16);
    R.silhouette[size_t(j) * R.silhouette_pitch + i] = uint8_t(id);
  }
  for (int k = tid; k < a.n_attach; k += blockDim.x) {  // the renderer-image records of the slots this renderer feeds
    const RenderAttachDev at = a.attach[k];
    if (at.renderer == r) {
      const RenderOutDev& o = a.out[r];
      const GeometryDev& G = a.geometry[at.body];
      const bool sil = at.slot == RS_REGION_SILHOUETTE || at.slot == RS_DEPTH_SILHOUETTE || at.slot == RS_TEXTURE_SILHOUETTE;
      RenderingDev d;
      d.image = sil ? R.silhouette : reinterpret_cast<const uint8_t*>(R.depth);
      d.image_size = S;
      d.pitch = sil ? R.silhouette_pitch : R.depth_pitch;
      d.corner_u = o.corner_u;
      d.corner_v = o.corner_v;
      d.scale = o.scale;
      d.projection_term_a = sil ? 0.0f : o.projection_term_a;
      d.projection_term_b = sil ? 0.0f : o.projection_term_b;
      d.id = sil ? (at.slot == RS_REGION_SILHOUETTE ? G.region_id : G.body_id) : 0;
      d.visible = a.visible[R.first_referenced + at.referenced_index];
      a.bodies[at.body].rend[at.slot] = d;
    }
  }
}

}  // namespace m3tb
