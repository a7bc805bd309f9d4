// C++ test of the reference-signature drop-in ORB_SLAM2::ORBextractor.
// Reads a raw 8-bit image, runs operator(), writes keypoints+descriptors for the Python side to compare with the oracle.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../self_commit_orb-slam2_b200/host/ORBextractor.h"

int main(int argc, char** argv) {
  if (argc < 5) return 2;
  const int w = atoi(argv[2]), h = atoi(argv[3]);
  b2s_cv::Mat img(h, w);
  FILE* f = fopen(argv[1], "rb");
  if (!f || fread(img.data, 1, (size_t)w * h, f) != (size_t)w * h) return 3;
  fclose(f);
  ORB_SLAM2::ORBextractor ex(1000, 1.2f, 8, 20, 7);
  std::vector<b2s_cv::KeyPoint> kps;
  b2s_cv::Mat desc, mask;
  ex(img, mask, kps, desc);
  if (ex.GetLevels() != 8 || ex.GetScaleFactors().size() != 8) return 4;
  if ((int)ex.mvImagePyramid.size() != 8 || ex.mvImagePyramid[0].cols != w) return 5;
  for (int i = 0; i < w * h; i += 977)
    if (ex.mvImagePyramid[0].data[i] != img.data[i]) return 6;  // level 0 is a copy of the input
  FILE* o = fopen(argv[4], "wb");
  int n = (int)kps.size();
  fwrite(&n, 4, 1, o);
  fwrite(kps.data(), sizeof(b2s_cv::KeyPoint), n, o);
  fwrite(desc.data, 32, n, o);
  fclose(o);
  // empty image: silent return, outputs untouched
  b2s_cv::Mat empty;
  std::vector<b2s_cv::KeyPoint> k2(3);
  ex(empty, mask, k2, desc);
  if (k2.size() != 3) return 7;
  printf("shim ok %d keypoints\n", n);
  return 0;
}
