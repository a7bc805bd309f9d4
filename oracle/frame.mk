# Builds the Frame checkers (test infrastructure), next to the oracle of Makefile:
#   _ref/libref_frame_seq.so    the reference's OWN src/Frame.cc, src/ORBextractor.cc and src/ORBmatcher.cc, compiled in
#                               place and unmodified like _ref/libref_frame_undistort.so (refshim_cv_undistort.h gives
#                               cv::undistortPoints), behind ref_frame_seq_glue.cpp (only where the reference's sources
#                               are present: REF)
#   _ref/libadapter_frame.so    the product's host/adapters/Frame_b200.cc and host/ORBextractor.cc in their place, behind
#                               the same glue, with the same flags and stand-ins, linking libb200slam.so (built first by
#                               build.py; skipped when it is absent).  refshim_cv.h alone: its cv::undistortPoints aborts.
#                               The drop-in ORBextractor.h is pre-included and the reference's header guard defined, as
#                               replacing include/ORBextractor.h does in the reference's own build (INTEGRATION.md §2).
# Every float expression is compiled as written: -ffp-contract=off.
# Used as `make -f frame.mk frame-ref REF=...`.
CXX ?= g++
PKG := ../self_commit_orb-slam2_b200
FRAME_FLAGS := -O2 -std=c++14 -ffp-contract=off -fPIC -shared -pthread -w -Wl,-Bsymbolic -DB2S_STUB_REAL_FRAME
FRAME_DBOW := $(REF)/Thirdparty/DBoW2/DBoW2/BowVector.cpp $(REF)/Thirdparty/DBoW2/DBoW2/FeatureVector.cpp
FRAME_DEPS := ref_frame_seq_glue.cpp refshim/refshim_cv.h refshim/slam_stubs.h

frame-ref: _ref/libref_frame_seq.so frame-adapters
_ref/libref_frame_seq.so: $(FRAME_DEPS) refshim/refshim_cv_undistort.h orb_undistort.cpp undistort_oracle.h orb_extract.cpp \
    orb_oracle.h
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(FRAME_FLAGS) -include refshim/refshim_cv_undistort.h -include refshim/slam_stubs.h -I refshim -I $(REF)/include \
	    -I $(REF) $(REF)/src/Frame.cc $(REF)/src/ORBextractor.cc $(REF)/src/ORBmatcher.cc $(FRAME_DBOW) ref_frame_seq_glue.cpp \
	    orb_extract.cpp orb_undistort.cpp -nostdlib++ -l:libstdc++.so.6 -o $@

ADAPTER_LIBS := $(if $(wildcard $(PKG)/libb200slam.so),_ref/libadapter_frame.so,)
frame-adapters: $(ADAPTER_LIBS)
_ref/libadapter_frame.so: $(FRAME_DEPS) $(PKG)/host/adapters/Frame_b200.cc $(PKG)/host/ORBextractor.cc \
    $(PKG)/host/ORBextractor.h $(PKG)/host/cv_compat.h $(PKG)/host/b2s_host.h ../include/b200slam.h $(PKG)/libb200slam.so
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(FRAME_FLAGS) -DB2S_HAVE_OPENCV -DB2S_ADAPTER_BUILD -DORBEXTRACTOR_H -include refshim/slam_stubs.h \
	    -include $(PKG)/host/ORBextractor.h -I refshim -I $(REF)/include -I $(REF) $(PKG)/host/adapters/Frame_b200.cc \
	    $(PKG)/host/ORBextractor.cc $(FRAME_DBOW) ref_frame_seq_glue.cpp -Wl,-z,defs -L$(PKG) -l:libb200slam.so \
	    -Wl,-rpath,'$$ORIGIN/../../self_commit_orb-slam2_b200' -nostdlib++ -l:libstdc++.so.6 -lm -o $@

.PHONY: frame-ref frame-adapters
