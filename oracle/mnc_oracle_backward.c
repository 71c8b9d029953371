/*
 * oracle/mnc_oracle_backward.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C CPU restatement of the backward passes of the reference's (daijifeng001/MNC) Caffe layers
 * ROIWarping, MaskResize, MaskPooling and ROIPooling (caffe-mnc/src/caffe/layers/
 * {roi_warping,mask_resize,mask_pooling,roi_pooling}_layer.cu), the companion of mnc_oracle.c's
 * forward restatements.  Only tests/ and scripts/ load this library (via oracle/oracle_backward.py);
 * mnc_b200/ never does.  Each function cites the reference file:line it follows and mirrors its
 * expressions term by term (same int/float/double promotions), compiled with -ffp-contract=off.
 * Pinned against the reference's own Backward_gpu compiled unmodified (oracle/backward.mk,
 * tests/test_ref_pin_backward.py): bit-exact against the -fmad=false build for every feature and
 * mask gradient.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>


/* ---------------------------------------------------------------------------------------
 * Backward passes of the four layers.  The argmax the reference's ROIWarping forward stores
 * (roi_warping_layer.cu:92-105: the clamped sample coordinate, or -1 for both axes when the sample
 * lies outside the map) is recomputed from the RoI geometry. */
static void warp_argmax(const float* roi, float spatial_scale, int H, int W, int ph_n, int pw_n,
                        int ph, int pw, float* ah, float* aw) {
  float roi_start_w = roundf(roi[1] * spatial_scale);
  float roi_start_h = roundf(roi[2] * spatial_scale);
  float roi_end_w = roundf(roi[3] * spatial_scale);
  float roi_end_h = roundf(roi[4] * spatial_scale);
  float roi_width = fmaxf(roi_end_w - roi_start_w, 0.f);
  float roi_height = fmaxf(roi_end_h - roi_start_h, 0.f);
  float bin_size_h = roi_height / (float)ph_n;
  float bin_size_w = roi_width / (float)pw_n;
  float h = roi_start_h + (float)ph * bin_size_h;
  float w = roi_start_w + (float)pw * bin_size_w;
  *ah = -1;
  *aw = -1;
  if (h < -0.5 || h > H - 0.5 || w < -0.5 || w > W - 0.5) return; /* :21-24 */
  if (h <= 0) h = 0;
  if (w <= 0) w = 0;
  if ((int)h >= H - 1) h = (float)(H - 1);
  if ((int)w >= W - 1) w = (float)(W - 1);
  *ah = h;
  *aw = w;
}

/* get_feature_gradient -- roi_warping_layer.cu:125-173 (getGradientWeight, mask_resize_layer.cu:
 * 86-133, is the same function). */
static float feature_gradient(float argmax_h, float argmax_w, int h, int w, int height, int width) {
  if (argmax_h < -0.5 || argmax_h > (height - 0.5) || argmax_w < -0.5 || argmax_w > (width - 0.5))
    return 0;
  if (argmax_h < 0) argmax_h = 0;
  if (argmax_w < 0) argmax_w = 0;
  int argmax_h_low = (int)argmax_h, argmax_w_low = (int)argmax_w, argmax_h_high, argmax_w_high;
  if (argmax_h_low >= height - 1) {
    argmax_h_high = argmax_h_low = height - 1;
    argmax_h = (float)argmax_h_low;
  } else
    argmax_h_high = argmax_h_low + 1;
  if (argmax_w_low >= width - 1) {
    argmax_w_high = argmax_w_low = width - 1;
    argmax_w = (float)argmax_w_low;
  } else
    argmax_w_high = argmax_w_low + 1;
  float weight = 0;
  if (h == argmax_h_low) {
    if (w == argmax_w_low)
      weight = (h + 1 - argmax_h) * (w + 1 - argmax_w);
    else if (w == argmax_w_high)
      weight = (h + 1 - argmax_h) * (argmax_w + 1 - w);
  } else if (h == argmax_h_high) {
    if (w == argmax_w_low)
      weight = (argmax_h + 1 - h) * (w + 1 - argmax_w);
    else if (w == argmax_w_high)
      weight = (argmax_h + 1 - h) * (argmax_w + 1 - w);
  }
  return weight;
}

/* get_coordinate_gradient -- roi_warping_layer.cu:247-304, float accumulators and weight, double
 * sub-expressions.  A sample outside the map (argmax -1) gives 0 here; the reference reads outside
 * the sampled plane there. */
static float coordinate_gradient(int coordinate_index, float h, float w, const float* data,
                                 float oh, float ow, int height, int width, int pooled_height,
                                 int pooled_width) {
  if (h == -1 && w == -1) return 0;
  int arg_interpolate_h = (int)h;
  int arg_interpolate_w = (int)w;
  if (arg_interpolate_h + 1 > height - 1 || arg_interpolate_w + 1 > width - 1) return 0;
  float map_ratio_h = (float)oh / (float)pooled_height;
  float map_ratio_w = (float)ow / (float)pooled_width;
  float weight = 0;
  int c1 = arg_interpolate_h * width + arg_interpolate_w;
  int c2 = arg_interpolate_h * width + (arg_interpolate_w + 1);
  int c3 = (arg_interpolate_h + 1) * width + arg_interpolate_w;
  int c4 = (arg_interpolate_h + 1) * width + (arg_interpolate_w + 1);
  float dxc = 0.0, dyc = 0.0, dw = 0.0, dh = 0.0;
  dxc += (-1.0 * (1.0 - h + arg_interpolate_h) * data[c1]);
  dxc += (1.0 * (1.0 - h + arg_interpolate_h) * data[c2]);
  dxc += (-1.0 * (h - arg_interpolate_h) * data[c3]);
  dxc += (1.0 * (h - arg_interpolate_h) * data[c4]);
  dyc += (-1.0 * (1.0 - w + arg_interpolate_w) * data[c1]);
  dyc += (-1.0 * (w - arg_interpolate_w) * data[c2]);
  dyc += (1.0 * (1.0 - w + arg_interpolate_w) * data[c3]);
  dyc += (1.0 * (w - arg_interpolate_w) * data[c4]);
  dw += ((0.5 - map_ratio_w) * (1.0 - h + arg_interpolate_h) * data[c1]);
  dw += ((-0.5 + map_ratio_w) * (1.0 - h + arg_interpolate_h) * data[c2]);
  dw += ((0.5 - map_ratio_w) * (h - arg_interpolate_h) * data[c3]);
  dw += ((-0.5 + map_ratio_w) * (h - arg_interpolate_h) * data[c4]);
  dh += ((0.5 - map_ratio_h) * (1.0 - w + arg_interpolate_w) * data[c1]);
  dh += ((0.5 - map_ratio_h) * (w - arg_interpolate_w) * data[c2]);
  dh += ((-0.5 + map_ratio_h) * (1.0 - w + arg_interpolate_w) * data[c3]);
  dh += ((-0.5 + map_ratio_h) * (w - arg_interpolate_w) * data[c4]);
  if (coordinate_index == 1)
    weight = 0.5 * dxc - dw;
  else if (coordinate_index == 2)
    weight = 0.5 * dyc - dh;
  else if (coordinate_index == 3)
    weight = 0.5 * dxc + dw;
  else if (coordinate_index == 4)
    weight = 0.5 * dyc + dh;
  return weight;
}

/* ROIWarping backward -- roi_warping_layer.cu:175-245 (feature), :306-361 + :409-434
 * (coordinates).  feat (B,C,H,W), rois (R,5), top_diff (R,C,ph,pw).  feat_diff (B,C,H,W) and
 * rois_diff (R,5) may each be NULL.  The coordinate terms are the reference's float buffer values;
 * their per-RoI sum is taken in double (the reference's thrust reduction order is unspecified).
 * rois_abs (R,5 doubles, may be NULL) receives the sums of the terms' magnitudes. */
void orc_roi_warp_backward(const float* feat, int B, int C, int H, int W, const float* rois, int R,
                           int ph_n, int pw_n, float spatial_scale, const float* top_diff,
                           float* feat_diff, float* rois_diff, double* rois_abs) {
  const int PP = ph_n * pw_n;
  float* amax_h = (float*)malloc(sizeof(float) * (size_t)(R > 0 ? R : 1) * PP);
  float* amax_w = (float*)malloc(sizeof(float) * (size_t)(R > 0 ? R : 1) * PP);
  for (int n = 0; n < R; ++n)
    for (int ph = 0; ph < ph_n; ++ph)
      for (int pw = 0; pw < pw_n; ++pw)
        warp_argmax(rois + 5 * n, spatial_scale, H, W, ph_n, pw_n, ph, pw,
                    amax_h + (size_t)n * PP + ph * pw_n + pw, amax_w + (size_t)n * PP + ph * pw_n + pw);
  if (feat_diff) {
#pragma omp parallel for schedule(dynamic, 1)
    for (int nc = 0; nc < B * C; ++nc) {
      const int n = nc / C, c = nc % C;
      for (int h = 0; h < H; ++h)
        for (int w = 0; w < W; ++w) {
          float gradient = 0;
          for (int roi_n = 0; roi_n < R; ++roi_n) {
            const float* r = rois + 5 * roi_n;
            int roi_level = (int)r[0];
            if (n != roi_level) continue;
            float roi_start_w = roundf(r[1] * spatial_scale);
            float roi_start_h = roundf(r[2] * spatial_scale);
            float roi_end_w = roundf(r[3] * spatial_scale);
            float roi_end_h = roundf(r[4] * spatial_scale);
            int in_roi = (w >= floorf(roi_start_w) && w <= ceilf(roi_end_w) &&
                          h >= floorf(roi_start_h) && h <= ceilf(roi_end_h));
            if (!in_roi) continue;
            size_t offset = ((size_t)roi_n * C + c) * PP;
            float roi_width = fmaxf(roi_end_w - roi_start_w + (float)1.0, (float)1.0);
            float roi_height = fmaxf(roi_end_h - roi_start_h + (float)1.0, (float)1.0);
            float bin_size_h = roi_height / (float)ph_n;
            float bin_size_w = roi_width / (float)pw_n;
            int phstart = (int)floorf((float)(h - roi_start_h - 1) / bin_size_h - 1);
            int phend = (int)ceilf((float)(h - roi_start_h + 1) / bin_size_h);
            int pwstart = (int)floorf((float)(w - roi_start_w - 1) / bin_size_w - 1);
            int pwend = (int)ceilf((float)(w - roi_start_w + 1) / bin_size_w);
            phstart = phstart < 0 ? 0 : (phstart > ph_n ? ph_n : phstart);
            phend = phend < 0 ? 0 : (phend > ph_n ? ph_n : phend);
            pwstart = pwstart < 0 ? 0 : (pwstart > pw_n ? pw_n : pwstart);
            pwend = pwend < 0 ? 0 : (pwend > pw_n ? pw_n : pwend);
            for (int ph = phstart; ph < phend; ++ph)
              for (int pw = pwstart; pw < pwend; ++pw) {
                int q = ph * pw_n + pw;
                float weight = feature_gradient(amax_h[(size_t)roi_n * PP + q],
                                                amax_w[(size_t)roi_n * PP + q], h, w, H, W);
                gradient += weight * top_diff[offset + q];
              }
          }
          feat_diff[(((size_t)n * C + c) * H + h) * W + w] = gradient;
        }
    }
  }
  if (rois_diff || rois_abs) {
#pragma omp parallel for schedule(dynamic, 1)
    for (int roi_n = 0; roi_n < R; ++roi_n) {
      const float* r = rois + 5 * roi_n;
      int roi_batch_ind = (int)r[0];
      int roi_start_w = (int)roundf(r[1] * spatial_scale);
      int roi_start_h = (int)roundf(r[2] * spatial_scale);
      int roi_end_w = (int)roundf(r[3] * spatial_scale);
      int roi_end_h = (int)roundf(r[4] * spatial_scale);
      int roi_width = roi_end_w - roi_start_w + 1 > 1 ? roi_end_w - roi_start_w + 1 : 1;
      int roi_height = roi_end_h - roi_start_h + 1 > 1 ? roi_end_h - roi_start_h + 1 : 1;
      float bin_size_h = (float)roi_height / (float)ph_n;
      float bin_size_w = (float)roi_width / (float)pw_n;
      double sum[5] = {0, 0, 0, 0, 0}, mag[5] = {0, 0, 0, 0, 0};
      if (roi_batch_ind >= 0 && roi_batch_ind < B) {
        for (int c = 0; c < C; ++c) {
          const float* data = feat + ((size_t)roi_batch_ind * C + c) * H * W;
          for (int q = 0; q < PP; ++q) {
            size_t offset = ((size_t)roi_n * C + c) * PP + q;
            float ih = amax_h[(size_t)roi_n * PP + q], iw = amax_w[(size_t)roi_n * PP + q];
            const float output_h = (ih - roi_start_h) / bin_size_h;
            const float output_w = (iw - roi_start_w) / bin_size_w;
            for (int k = 1; k < 5; ++k) {
              float weight = spatial_scale * coordinate_gradient(k, ih, iw, data, output_h, output_w,
                                                                 H, W, ph_n, pw_n);
              float term = weight * top_diff[offset];
              sum[k] += term;
              mag[k] += fabs(term);
            }
          }
        }
      }
      for (int k = 0; k < 5; ++k) {
        if (rois_diff) rois_diff[5 * roi_n + k] = (float)sum[k];
        if (rois_abs) rois_abs[5 * roi_n + k] = mag[k];
      }
    }
  }
  free(amax_h);
  free(amax_w);
}

/* MaskResize backward -- mask_resize_layer.cu:135-173.  top_diff (N,C,oh,ow) -> in_diff
 * (N,C,ih,iw).  The reference may read top_diff one element past a row, or past the plane, where
 * the weight is 0 (the sample lies at >= dim - 0.5); such terms are not read here. */
void orc_mask_resize_backward(const float* top_diff, int N, int C, int ih_n, int iw_n, int oh_n,
                              int ow_n, float* in_diff) {
  float ratio_h = (float)ih_n / (float)oh_n;
  float ratio_w = (float)iw_n / (float)ow_n;
#pragma omp parallel for
  for (int nc = 0; nc < N * C; ++nc) {
    const float* offset_top_diff = top_diff + (size_t)nc * oh_n * ow_n;
    for (int h = 0; h < ih_n; ++h)
      for (int w = 0; w < iw_n; ++w) {
        float gradient = 0.0;
        float map_x = (float)w / ratio_w;
        float map_y = (float)h / ratio_h;
        int output_h_start = (int)floorf(map_y);
        int output_w_start = (int)floorf(map_x);
        for (int ph = output_h_start; ph <= output_h_start + 1; ++ph)
          for (int pw = output_w_start; pw <= output_w_start + 1; ++pw) {
            float iw = (float)pw * ratio_w;
            float ih = (float)ph * ratio_h;
            if (fabsf(iw - w) >= 1 || fabsf(ih - h) >= 1) continue;
            float weight = feature_gradient(ih, iw, h, w, ih_n, iw_n);
            if (ph >= oh_n || pw >= ow_n) continue; /* weight is 0 there */
            gradient += weight * offset_top_diff[ph * ow_n + pw];
          }
        in_diff[((size_t)nc * ih_n + h) * iw_n + w] = gradient;
      }
  }
}

/* MaskPooling backward -- mask_pooling_layer.cu:43-76.  feat_diff / mask_diff may be NULL. */
void orc_mask_pool_backward(const float* feat, const float* mask, const float* top_diff, int N,
                            int C, int H, int W, float* feat_diff, float* mask_diff) {
  const size_t hw = (size_t)H * W;
#pragma omp parallel for
  for (int n = 0; n < N; ++n) {
    if (feat_diff)
      for (int c = 0; c < C; ++c)
        for (size_t i = 0; i < hw; ++i)
          feat_diff[((size_t)n * C + c) * hw + i] = top_diff[((size_t)n * C + c) * hw + i] * mask[n * hw + i];
    if (mask_diff)
      for (size_t i = 0; i < hw; ++i) {
        float gradient = 0.0;
        for (int c = 0; c < C; ++c)
          gradient += top_diff[((size_t)n * C + c) * hw + i] * feat[((size_t)n * C + c) * hw + i];
        mask_diff[n * hw + i] = gradient;
      }
  }
}

/* ROIPooling backward -- roi_pooling_layer.cu:94-165.  top_diff / argmax (R,C,ph,pw) ->
 * feat_diff (B,C,H,W). */
void orc_roi_pool_backward(const float* top_diff, const int* argmax, int B, int C, int H, int W,
                           const float* rois, int R, int ph_n, int pw_n, float spatial_scale,
                           float* feat_diff) {
#pragma omp parallel for schedule(dynamic, 1)
  for (int nc = 0; nc < B * C; ++nc) {
    const int n = nc / C, c = nc % C;
    for (int h = 0; h < H; ++h)
      for (int w = 0; w < W; ++w) {
        float gradient = 0;
        for (int roi_n = 0; roi_n < R; ++roi_n) {
          const float* r = rois + 5 * roi_n;
          int roi_batch_ind = (int)r[0];
          if (n != roi_batch_ind) continue;
          int roi_start_w = (int)roundf(r[1] * spatial_scale);
          int roi_start_h = (int)roundf(r[2] * spatial_scale);
          int roi_end_w = (int)roundf(r[3] * spatial_scale);
          int roi_end_h = (int)roundf(r[4] * spatial_scale);
          int in_roi = (w >= roi_start_w && w <= roi_end_w && h >= roi_start_h && h <= roi_end_h);
          if (!in_roi) continue;
          size_t offset = ((size_t)roi_n * C + c) * ph_n * pw_n;
          int roi_width = roi_end_w - roi_start_w + 1 > 1 ? roi_end_w - roi_start_w + 1 : 1;
          int roi_height = roi_end_h - roi_start_h + 1 > 1 ? roi_end_h - roi_start_h + 1 : 1;
          float bin_size_h = (float)roi_height / (float)ph_n;
          float bin_size_w = (float)roi_width / (float)pw_n;
          int phstart = (int)floorf((float)(h - roi_start_h) / bin_size_h);
          int phend = (int)ceilf((float)(h - roi_start_h + 1) / bin_size_h);
          int pwstart = (int)floorf((float)(w - roi_start_w) / bin_size_w);
          int pwend = (int)ceilf((float)(w - roi_start_w + 1) / bin_size_w);
          phstart = phstart < 0 ? 0 : (phstart > ph_n ? ph_n : phstart);
          phend = phend < 0 ? 0 : (phend > ph_n ? ph_n : phend);
          pwstart = pwstart < 0 ? 0 : (pwstart > pw_n ? pw_n : pwstart);
          pwend = pwend < 0 ? 0 : (pwend > pw_n ? pw_n : pwend);
          for (int ph = phstart; ph < phend; ++ph)
            for (int pw = pwstart; pw < pwend; ++pw)
              if (argmax[offset + ph * pw_n + pw] == (h * W + w))
                gradient += top_diff[offset + ph * pw_n + pw];
        }
        feat_diff[(((size_t)n * C + c) * H + h) * W + w] = gradient;
      }
  }
}
