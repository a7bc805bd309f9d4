// LocalMapping::KeyFrameCulling over b2s_keyframe_culling, and ProcessNewKeyFrame's association with MapPointCulling over
// b2s_process_new_keyframe, against the reference's unchanged include/KeyFrame.h, include/MapPoint.h and include/Map.h.
#ifndef B2S_LOCALMAPPING_B200_H
#define B2S_LOCALMAPPING_B200_H

#include <list>

#include "KeyFrame.h"
#include "Map.h"

namespace ORB_SLAM2 {
namespace b200 {

// Does what LocalMapping::KeyFrameCulling (src/LocalMapping.cc:873-956) does with mpCurrentKeyFrame = pCurrentKF and
// mbMonocular = bMonocular: the verdicts come from one device call, then the reference's own KeyFrame::SetBadFlag runs
// on the culled and deferred keyframes in list order, so the spanning tree, the connections and the map / database
// erasure are the reference's.  Returns 0, or a B2S_ERR_* code with the graph unchanged.
int KeyFrameCulling(KeyFrame* pCurrentKF, bool bMonocular);

// Does what LocalMapping::ProcessNewKeyFrame (src/LocalMapping.cc:217-253) after ComputeBoW, then MapPointCulling
// (:261-308), do with mpCurrentKeyFrame = pKF, mpMap = pMap, mlpRecentAddedMapPoints = lRecent and mbMonocular =
// bMonocular: the association, UpdateNormalAndDepth, ComputeDistinctiveDescriptors and the culling verdicts come from
// one device call; the reference's own AddObservation, UpdateConnections, Map::AddKeyFrame and MapPoint::SetBadFlag
// apply them in the reference's order, and lRecent is rewritten.  Returns 0, or a B2S_ERR_* code with the graph
// unchanged.
int ProcessNewKeyFrame(KeyFrame* pKF, Map* pMap, std::list<MapPoint*>& lRecent, bool bMonocular);

}  // namespace b200
}  // namespace ORB_SLAM2
#endif
