# Builds the OptimizeSim3 checkers (test infrastructure), next to the oracle of Makefile:
#   liborb_sim3opt.so          the CPU restatement (sim3opt.cpp, with the essential graph oracle's Sim3 operations)
#   _ref/libref_sim3opt.so     the reference's OWN src/Optimizer.cc + src/Converter.cc + the whole vendored g2o (the
#                              objects Makefile builds for libref_optimizer.so) behind ref_sim3opt_glue.cpp (only where
#                              the reference's sources are present: REF)
#   _ref/libadapter_sim3opt.so the product's drop-in host/adapters/Optimizer_b200.cc behind the same glue (needs
#                              libb200slam.so, built first by build.py)
# Used as `make -f sim3opt.mk liborb_sim3opt.so` and `make -f sim3opt.mk sim3opt-ref REF=...` (after `make ref REF=...`).
include Makefile

liborb_sim3opt.so: sim3opt.cpp essential.cpp sim3opt_oracle.h essential_oracle.h
	$(CXX) $(CXXFLAGS) -shared -o $@ sim3opt.cpp essential.cpp

sim3opt-ref: _ref/libref_sim3opt.so sim3opt-adapters
_ref/obj/ref_sim3opt_glue.o: ref_sim3opt_glue.cpp sim3opt_oracle.h essential_oracle.h refshim/eigen/refshim_eigen.h \
    refshim/slam_stubs_optimizer.h refshim/refshim_cv.h
	$(if $(REF),,$(error set REF to the reference's source tree))
	@mkdir -p $(dir $@)
	$(CXX) $(OPT_FLAGS) -include refshim/slam_stubs_optimizer.h -I . -I $(REF)/include -I $(REF) -c $< -o $@
_ref/libref_sim3opt.so: $(G2O_OBJS) _ref/obj/Optimizer.o _ref/obj/Converter.o _ref/obj/ref_sim3opt_glue.o
	$(CXX) -shared -pthread -Wl,-Bsymbolic -o $@ $^

S3O_ADAPTER_LIBS := $(if $(wildcard $(PKG)/libb200slam.so),_ref/libadapter_sim3opt.so,)
sim3opt-adapters: $(S3O_ADAPTER_LIBS)
_ref/libadapter_sim3opt.so: $(PKG)/host/adapters/Optimizer_b200.cc ref_sim3opt_glue.cpp sim3opt_oracle.h \
    essential_oracle.h refshim/eigen/refshim_eigen.h refshim/slam_stubs_optimizer.h refshim/refshim_cv.h \
    ../include/b200slam.h $(PKG)/libb200slam.so
	$(if $(REF),,$(error set REF to the reference's source tree))
	mkdir -p _ref
	$(CXX) $(OPT_FLAGS) -DB2S_ADAPTER_BUILD -shared -Wl,-Bsymbolic -include refshim/slam_stubs_optimizer.h -I . -I ../include \
	    -I $(REF)/include -I $(REF) $(PKG)/host/adapters/Optimizer_b200.cc ref_sim3opt_glue.cpp \
	    -L$(PKG) -l:libb200slam.so -Wl,-rpath,'$$ORIGIN/../../self_commit_orb-slam2_b200' -o $@

.PHONY: sim3opt-ref sim3opt-adapters
