// Compile check of the toROSMsg wrapper of m-loam_b200/host/mloam_adapter.hpp against the stub headers, with the messages of
// lidar_mapper_keyframe.cpp:690-714 and :780-851.  Compiled, never run: the calls need an H100.
#include <Eigen/Dense>
#include <ceres/ceres.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>
#include <sensor_msgs/PointCloud2.h>

#include "common/types/type.h"
#include "reference_types.h"

#include "../../m-loam_b200/host/mloam_adapter.hpp"

int adapter_cloud_msgs_use(mloam_ctx_t *ctx) {
  sensor_msgs::PointCloud2 laser_cloud_full_res_msg, laser_cloud_surf_last_msg, laser_cloud_corner_last_msg, laser_cloud_surround_msg,
      laser_cloud_map_msg;
  mloam::toROSMsg(ctx, {MLOAM_MSG_FULL_RES, MLOAM_MSG_SURF_LAST, MLOAM_MSG_CORNER_LAST},
                  {&laser_cloud_full_res_msg, &laser_cloud_surf_last_msg, &laser_cloud_corner_last_msg});
  mloam::toROSMsg(ctx, MLOAM_MSG_SURROUND, laser_cloud_surround_msg);
  mloam::toROSMsg(ctx, MLOAM_MSG_GLOBAL_MAP0, laser_cloud_map_msg);
  laser_cloud_map_msg.header.frame_id = "/world";
  return (int)(laser_cloud_full_res_msg.width + laser_cloud_surround_msg.data.size() + laser_cloud_map_msg.fields.size());
}
