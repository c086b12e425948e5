# oracle/ctxlib_ref.mk -- TEST INFRASTRUCTURE, not product code.
#
# The reference's context-library engine as oracle/_ref/libhhref_ctxlib.so: oracle/ctxlib_shim.cpp linked against the
# reference objects of oracle/ref_build.mk (same sources, same flags), with the reference's data/context_data.lib
# embedded by `ld -r -b binary` the way ref_build.mk embeds context_data.crf.
#
# Usage:  make -f oracle/ctxlib_ref.mk -j8        (from the repo root, after or instead of oracle/ref_build.mk)
include oracle/ref_build.mk

.DEFAULT_GOAL := ctxlib

ctxlib: $(OUT)/libhhref_ctxlib.so

$(OUT)/obj/res_lib.o: $(OUT)/gen/.stamp
	cd $(REF)/data && ld -r -b binary -o $(abspath $@) context_data.lib

$(OUT)/libhhref_ctxlib.so: oracle/ctxlib_shim.cpp $(OUT)/libhhref.a $(OUT)/obj/res_lib.o
	$(CXX) $(CXXFLAGS) $(INC) -shared -o $@ oracle/ctxlib_shim.cpp $(OUT)/obj/res_lib.o \
	    -Wl,--whole-archive $(OUT)/libhhref.a -Wl,--no-whole-archive -lgomp
