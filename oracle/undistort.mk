# Builds the undistortion / RGB-D depth checkers (test infrastructure), next to the oracle of Makefile:
#   liborb_undistort.so               the CPU restatement of cv::undistortPoints (orb_undistort.cpp)
#   _ref/libref_frame_undistort.so    the reference's OWN src/Frame.cc (with its ORBextractor.cc and ORBmatcher.cc), compiled
#                                     in place and unmodified like _ref/libref_frame.so, but against
#                                     refshim/refshim_cv_undistort.h, whose cv::undistortPoints is the restatement; behind
#                                     ref_frame_undistort_glue.cpp, which builds the monocular and RGB-D Frames (only where
#                                     the reference's sources are present: REF)
# Every float expression is compiled as written: -ffp-contract=off.
# Used as `make -f undistort.mk liborb_undistort.so` and `make -f undistort.mk undistort-ref REF=...`.
CXX ?= g++
UND_DEPS := ref_frame_undistort_glue.cpp orb_undistort.cpp undistort_oracle.h refshim/refshim_cv_undistort.h \
    refshim/refshim_cv.h refshim/slam_stubs.h orb_extract.cpp orb_oracle.h

liborb_undistort.so: orb_undistort.cpp undistort_oracle.h
	$(CXX) -O3 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -std=c++17 -fPIC -Wall -shared -o $@ orb_undistort.cpp

undistort-ref: _ref/libref_frame_undistort.so
_ref/libref_frame_undistort.so: $(UND_DEPS)
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) -O2 -std=c++14 -ffp-contract=off -fPIC -shared -pthread -w -Wl,-Bsymbolic -DB2S_STUB_REAL_FRAME \
	    -include refshim/refshim_cv_undistort.h -include refshim/slam_stubs.h -I refshim -I $(REF)/include -I $(REF) \
	    $(REF)/src/Frame.cc $(REF)/src/ORBextractor.cc $(REF)/src/ORBmatcher.cc $(REF)/Thirdparty/DBoW2/DBoW2/BowVector.cpp \
	    $(REF)/Thirdparty/DBoW2/DBoW2/FeatureVector.cpp ref_frame_undistort_glue.cpp orb_extract.cpp orb_undistort.cpp \
	    -nostdlib++ -l:libstdc++.so.6 -o $@

.PHONY: undistort-ref
