# Builds the global bundle adjustment checkers (test infrastructure), next to the oracle of Makefile:
#   liborb_gba.so          the CPU restatement (gba.cpp, which compiles local_ba.cpp's struct BA into it)
#   _ref/libref_gba.so     the reference's OWN src/Optimizer.cc + src/Converter.cc + the whole vendored g2o (the objects
#                          Makefile builds for libref_optimizer.so) behind ref_gba_glue.cpp (only where the reference's
#                          sources are present: REF)
#   _ref/libadapter_gba.so the product's drop-in host/adapters/Optimizer_b200.cc behind the same glue (needs
#                          libb200slam.so, built first by build.py)
# Used as `make -f gba.mk liborb_gba.so` and `make -f gba.mk gba-ref REF=...` (after `make ref REF=...`).
include Makefile

liborb_gba.so: gba.cpp gba_oracle.h local_ba.cpp orb_oracle.h
	$(CXX) $(CXXFLAGS) -shared -o $@ gba.cpp

gba-ref: _ref/libref_gba.so gba-adapters
_ref/obj/ref_gba_glue.o: ref_gba_glue.cpp gba_oracle.h orb_oracle.h refshim/eigen/refshim_eigen.h refshim/slam_stubs_optimizer.h \
    refshim/refshim_cv.h
	$(if $(REF),,$(error set REF to the reference's source tree))
	@mkdir -p $(dir $@)
	$(CXX) $(OPT_FLAGS) -include refshim/slam_stubs_optimizer.h -I . -I $(REF)/include -I $(REF) -c $< -o $@
_ref/libref_gba.so: $(G2O_OBJS) _ref/obj/Optimizer.o _ref/obj/Converter.o _ref/obj/ref_gba_glue.o
	$(CXX) -shared -pthread -Wl,-Bsymbolic -o $@ $^

GBA_ADAPTER_LIBS := $(if $(wildcard $(PKG)/libb200slam.so),_ref/libadapter_gba.so,)
gba-adapters: $(GBA_ADAPTER_LIBS)
_ref/libadapter_gba.so: $(PKG)/host/adapters/Optimizer_b200.cc ref_gba_glue.cpp gba_oracle.h orb_oracle.h \
    refshim/eigen/refshim_eigen.h refshim/slam_stubs_optimizer.h refshim/refshim_cv.h ../include/b200slam.h $(PKG)/libb200slam.so
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(OPT_FLAGS) -DB2S_ADAPTER_BUILD -shared -Wl,-Bsymbolic -include refshim/slam_stubs_optimizer.h -I . -I ../include \
	    -I $(REF)/include -I $(REF) $(PKG)/host/adapters/Optimizer_b200.cc ref_gba_glue.cpp \
	    -L$(PKG) -l:libb200slam.so -Wl,-rpath,'$$ORIGIN/../../self_commit_orb-slam2_b200' -o $@

.PHONY: gba-ref gba-adapters
