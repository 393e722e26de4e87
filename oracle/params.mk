# ORACLE build recipe (test infrastructure) for pafprocess with other constants than the reference's
# (oracle/post_params.py runs it; tests/test_post_params_host.py compares against its products).
#   make -f params.mk port     the parameterised plain-C port, libpafprocess_params.so
#   make -f params.mk ref-set SET=<name> PAF_THRESH=.. PAF_SAMPLES=.. PAF_MIN_ABOVE=.. MIN_PARTS=.. MIN_PERSON_SCORE=..
#                              the reference's own pafprocess.cpp compiled with those five constants, as
#                              _ref/<name>/libpafprocess_ref.so (git-ignored, travels to the GPU box with the snapshot)
# The reference's pafprocess.h is copied to _ref/<name>/ with the five constants substituted (the copy is rewritten only
# when its text changes, so the .so is rebuilt exactly when the values change).  The .cpp is read from stdin: compiled
# where it lies, its quoted #include "pafprocess.h" would find the unmodified header beside it before any -I directory.
REF ?= /root/reference
CC ?= gcc
CXX ?= g++
SRC = $(REF)/lib/pafprocess
SETDIR = _ref/$(SET)

port: libpafprocess_params.so

libpafprocess_params.so: pafprocess_params.c pafprocess_port.c
	$(CC) -O2 -ffp-contract=off -shared -fPIC $< -o $@ -lm -lpthread

ref-set: $(SETDIR)/libpafprocess_ref.so

.PHONY: port ref-set FORCE
FORCE:

$(SETDIR)/pafprocess.h: $(SRC)/pafprocess.h FORCE
	@test -n "$(SET)" -a -n "$(PAF_THRESH)" -a -n "$(PAF_SAMPLES)" -a -n "$(PAF_MIN_ABOVE)" -a -n "$(MIN_PARTS)" \
	    -a -n "$(MIN_PERSON_SCORE)" || { echo "ref-set needs SET and the five values" >&2; exit 1; }
	mkdir -p $(SETDIR)
	sed -e 's/^const float THRESH_VECTOR_SCORE = .*;$$/const float THRESH_VECTOR_SCORE = $(PAF_THRESH);/' \
	    -e 's/^const int STEP_PAF = .*;$$/const int STEP_PAF = $(PAF_SAMPLES);/' \
	    -e 's/^const int THRESH_VECTOR_CNT1 = .*;$$/const int THRESH_VECTOR_CNT1 = $(PAF_MIN_ABOVE);/' \
	    -e 's/^const int THRESH_PART_CNT = .*;$$/const int THRESH_PART_CNT = $(MIN_PARTS);/' \
	    -e 's/^const float THRESH_HUMAN_SCORE = .*;$$/const float THRESH_HUMAN_SCORE = $(MIN_PERSON_SCORE);/' \
	    $(SRC)/pafprocess.h > $@.tmp
	test `grep -cxF -e 'const float THRESH_VECTOR_SCORE = $(PAF_THRESH);' -e 'const int STEP_PAF = $(PAF_SAMPLES);' \
	    -e 'const int THRESH_VECTOR_CNT1 = $(PAF_MIN_ABOVE);' -e 'const int THRESH_PART_CNT = $(MIN_PARTS);' \
	    -e 'const float THRESH_HUMAN_SCORE = $(MIN_PERSON_SCORE);' $@.tmp` -eq 5
	cmp -s $@.tmp $@ && rm -f $@.tmp || mv -f $@.tmp $@

$(SETDIR)/libpafprocess_ref.so: $(SETDIR)/pafprocess.h ref_shim.cpp $(SRC)/pafprocess.cpp
	$(CXX) -O2 -shared -fPIC -I$(SETDIR) -x c++ - -x none ref_shim.cpp -o $@ < $(SRC)/pafprocess.cpp
