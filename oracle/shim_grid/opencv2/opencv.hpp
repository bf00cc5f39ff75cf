// oracle/shim_grid/opencv2/opencv.hpp — NOT OpenCV: the stand-ins of oracle/shim/opencv2 plus what src/a_star.cpp and
// src/dijkstra.cpp also use, cv::Point and cv::rectangle.  oracle/grid.mk puts this directory ahead of oracle/shim, so
// the planners' <opencv2/opencv.hpp> resolves here while <opencv2/core/core.hpp> and <opencv2/highgui/highgui.hpp>
// resolve to oracle/shim (whose copy of opencv.hpp is then already included).
//
// Unlike the other stand-ins, cv::rectangle runs: the planners call it from inside the search, and it hands each
// call's corners, colour and thickness to rectangle_recorder() when one is set (null by default), so that
// oracle/shim_grid/ref_wrap_grid.cpp can recover the obstacle map, the expansion trace and the path from the calls.
#ifndef CRB_SHIM_GRID_OPENCV_
#define CRB_SHIM_GRID_OPENCV_
#include "../../shim/opencv2/opencv.hpp"
namespace cv {
typedef Point2i Point;
typedef void (*RectangleRecorder)(int x1, int y1, int x2, int y2, const Scalar& color, int thickness);
inline RectangleRecorder& rectangle_recorder() {
  static RectangleRecorder r = 0;
  return r;
}
inline void rectangle(const Mat&, Point2i a, Point2i b, const Scalar& color, int thickness = 1) {
  if (rectangle_recorder()) rectangle_recorder()(a.x, a.y, b.x, b.y, color, thickness);
}
}  // namespace cv
#endif
