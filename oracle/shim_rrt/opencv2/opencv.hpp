// oracle/shim_rrt/opencv2/opencv.hpp — NOT OpenCV: the stand-ins of oracle/shim/opencv2 plus what include/rrt.h also
// uses, cv::Point.  oracle/Makefile puts this directory ahead of oracle/shim, so the header's <opencv2/opencv.hpp>
// resolves here while <opencv2/core/core.hpp> and <opencv2/highgui/highgui.hpp> resolve to oracle/shim.
//
// RRT::planning loops until it reaches the goal and draws one cv::line per accepted node.  cv::Point is a type of its
// own so that the cv::line below, which takes it, is a better match than shim/'s: it counts its calls and throws
// cv::LineLimit once line_limit() of them are exceeded, which bounds a run that would otherwise never end.
#ifndef CRB_SHIM_RRT_OPENCV_
#define CRB_SHIM_RRT_OPENCV_
#include "../../shim/opencv2/opencv.hpp"
namespace cv {
struct Point : Point2i {
  Point(int a, int b) : Point2i(a, b) {}
};
struct LineLimit {};
inline long& line_count() {
  static long c = 0;
  return c;
}
inline long& line_limit() {
  static long l = 0;
  return l;
}
inline void line(Mat&, const Point&, const Point&, const Scalar&, int = 1) {
  if (++line_count() > line_limit()) throw LineLimit();
}
}  // namespace cv
#endif
