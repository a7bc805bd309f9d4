# Builds the covisibility-update checkers (test infrastructure), next to the oracle of Makefile:
#   liborb_covis.so           the CPU restatement (covis.cpp)
#   _ref/libref_keyframe.so   the reference's OWN src/KeyFrame.cc, compiled in place and unmodified with its include/KeyFrame.h
#                             and include/Frame.h, against the stand-ins of refshim/slam_stubs_keyframe.h (only where the
#                             reference's sources are present: REF)
#   _ref/libadapter_covis.so  the product's host/adapters/Covisibility_b200.cc behind the same glue (needs libb200slam.so,
#                             built first by build.py)
# Used as `make -f covis.mk liborb_covis.so` and `make -f covis.mk covis-ref REF=...`.
CXX ?= g++
PKG := ../self_commit_orb-slam2_b200
COVIS_FLAGS := -O2 -std=c++14 -fPIC -shared -pthread -w -Wl,-Bsymbolic -include refshim/slam_stubs_keyframe.h \
    -I refshim/keyframe -I refshim -I ../include -I $(REF)/include -I $(REF)
# sim3solver.cpp / init.cpp: the cv2-pinned matrix primitives behind the cv stand-in's expressions (SetPose)
COVIS_DBOW := sim3solver.cpp init.cpp $(REF)/Thirdparty/DBoW2/DBoW2/BowVector.cpp \
    $(REF)/Thirdparty/DBoW2/DBoW2/FeatureVector.cpp -lm -nostdlib++ -l:libstdc++.so.6

liborb_covis.so: covis.cpp ../include/b200slam.h
	$(CXX) -O3 -march=x86-64-v3 -std=c++17 -fPIC -Wall -shared -o $@ covis.cpp

covis-ref: _ref/libref_keyframe.so covis-adapters
_ref/libref_keyframe.so: ref_covis_glue.cpp refshim/slam_stubs_keyframe.h refshim/refshim_cv_keyframe.h ../include/b200slam.h \
    sim3solver.cpp init.cpp
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(COVIS_FLAGS) $(REF)/src/KeyFrame.cc ref_covis_glue.cpp $(COVIS_DBOW) -o $@

ADAPTER_LIBS := $(if $(wildcard $(PKG)/libb200slam.so),_ref/libadapter_covis.so,)
covis-adapters: $(ADAPTER_LIBS)
_ref/libadapter_covis.so: $(PKG)/host/adapters/Covisibility_b200.cc $(PKG)/host/adapters/Covisibility_b200.h \
    ref_covis_glue.cpp refshim/slam_stubs_keyframe.h ../include/b200slam.h $(PKG)/libb200slam.so
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(COVIS_FLAGS) -DB2S_ADAPTER_BUILD -I $(PKG)/host $(REF)/src/KeyFrame.cc $(PKG)/host/adapters/Covisibility_b200.cc \
	    ref_covis_glue.cpp $(COVIS_DBOW) -L$(PKG) -l:libb200slam.so -Wl,-rpath,'$$ORIGIN/../../self_commit_orb-slam2_b200' -o $@

.PHONY: covis-ref covis-adapters
