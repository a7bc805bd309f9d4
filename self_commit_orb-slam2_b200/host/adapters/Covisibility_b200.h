// Batched KeyFrame::UpdateConnections over b2s_update_connections, against the reference's unchanged include/KeyFrame.h.
#ifndef B2S_COVISIBILITY_B200_H
#define B2S_COVISIBILITY_B200_H

#include <map>
#include <vector>

#include "KeyFrame.h"

namespace ORB_SLAM2 {
namespace b200 {

// What a caller of the one-at-a-time reference reads around each call, per member in call order:
// GetVectorCovisibleKeyFrames() just before the call and the connection map (GetConnectedKeyFrames()' keys, with
// weights) just after it.
struct CovisibilityReads {
  std::vector<std::vector<KeyFrame*> > before;
  std::vector<std::map<KeyFrame*, int> > after;
};

// Calls UpdateConnections on vpKFs in order (repeats allowed) as one device call.  The graph ends in the state the
// reference's calls one after another leave when the keyframes' address order is their mnId order (DESIGN §2).
// Returns 0, or a B2S_ERR_* code with the graph unchanged.
int UpdateConnections(const std::vector<KeyFrame*>& vpKFs, CovisibilityReads* reads);

}  // namespace b200
}  // namespace ORB_SLAM2
#endif
