// LocalMapping::KeyFrameCulling over b2s_keyframe_culling, against the reference's unchanged include/KeyFrame.h and
// include/MapPoint.h.
#ifndef B2S_LOCALMAPPING_B200_H
#define B2S_LOCALMAPPING_B200_H

#include "KeyFrame.h"

namespace ORB_SLAM2 {
namespace b200 {

// Does what LocalMapping::KeyFrameCulling (src/LocalMapping.cc:873-956) does with mpCurrentKeyFrame = pCurrentKF and
// mbMonocular = bMonocular: the verdicts come from one device call, then the reference's own KeyFrame::SetBadFlag runs
// on the culled and deferred keyframes in list order, so the spanning tree, the connections and the map / database
// erasure are the reference's.  Returns 0, or a B2S_ERR_* code with the graph unchanged.
int KeyFrameCulling(KeyFrame* pCurrentKF, bool bMonocular);

}  // namespace b200
}  // namespace ORB_SLAM2
#endif
