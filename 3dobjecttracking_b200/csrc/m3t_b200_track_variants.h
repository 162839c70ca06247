// m3t_b200_track_variants.h - the k_track instantiations of libm3t_b200.so. Each group is compiled in its own
// translation unit (m3t_b200_track_<g>.cu) so that nvcc -t builds them in parallel; m3t_b200.cu only declares them.
#pragma once
#define M3TB_TRACK_GROUP_0(X) \
  X(256, 1, true, false) \
  X(512, 1, true, false) \
  X(512, 2, true, false) \
  X(512, 4, true, false)
#define M3TB_TRACK_GROUP_1(X) \
  X(256, 1, true, true) \
  X(512, 1, true, true) \
  X(512, 2, true, true) \
  X(512, 4, true, true)
#define M3TB_TRACK_GROUP_2(X) \
  X(256, 1, false, false) \
  X(512, 1, false, false) \
  X(512, 2, false, false) \
  X(512, 4, false, false)
#define M3TB_TRACK_GROUP_3(X) \
  X(256, 1, false, true) \
  X(512, 1, false, true) \
  X(512, 2, false, true) \
  X(512, 4, false, true)
#define M3TB_TRACK_ALL(X) M3TB_TRACK_GROUP_0(X) M3TB_TRACK_GROUP_1(X) M3TB_TRACK_GROUP_2(X) M3TB_TRACK_GROUP_3(X)
