# oracle/cli.mk -- builds _ref/lz4, a CHECKER (test infrastructure), never the product: the reference's upstream
# command-line tool (orig/programs/lz4cli.c, lz4io.c, bench.c, datagen.c over the four lib sources), compiled from
# where they lie under $(REF).  It is the oracle of how `lz4 -d` reads whole .lz4 inputs (concatenated, skippable and
# legacy members, its error numbers).  No reference source is written to disk; only the binary lands in _ref/.
# Nothing is done where $(REF) is absent.
#   make -C oracle -f cli.mk
REF ?= /root/reference
CC ?= gcc
CLIFLAGS ?= -O2

cli:
	@if [ -f $(REF)/orig/programs/lz4cli.c ]; then \
	  mkdir -p _ref && \
	  $(CC) $(CLIFLAGS) -I$(REF)/orig/lib -o _ref/lz4 \
	      $(REF)/orig/programs/lz4cli.c $(REF)/orig/programs/lz4io.c $(REF)/orig/programs/bench.c \
	      $(REF)/orig/programs/datagen.c $(REF)/orig/lib/lz4.c $(REF)/orig/lib/lz4hc.c \
	      $(REF)/orig/lib/lz4frame.c $(REF)/orig/lib/xxhash.c && \
	  echo "built _ref/lz4"; \
	else echo "reference not present: keeping prebuilt _ref/lz4 (if any)"; fi

.PHONY: cli
