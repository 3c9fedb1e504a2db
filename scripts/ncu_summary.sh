#!/bin/bash
# Extract the judged metrics of an .ncu-rep into profiles/<name>.ncu-summary.csv (run where ncu is installed).
# usage: scripts/ncu_summary.sh prof_x.ncu-rep [more.ncu-rep ...]
METRICS='Kernel Name|gpu__time_duration.sum|dram__bytes_read.sum$|dram__bytes_write.sum$|gpu__dram_throughput.avg.pct|lts__t_sector_hit_rate.pct|sm__warps_active.avg.pct|launch__registers_per_thread$|launch__grid_size|launch__block_size|launch__occupancy_limit|smsp__issue_active.avg.pct|sm__throughput.avg.pct|l1tex__throughput.avg.pct_of_peak_sustained_elapsed|lts__throughput.avg.pct|sm__pipe_tensor|smsp__average_warps_issue_stalled_(long_scoreboard|lg_throttle|barrier|membar|short_scoreboard)_per_issue_active|launch__shared_mem_per_block|launch__waves|nvlrx__bytes.sum$|nvltx__bytes.sum$|lts__t_bytes.sum$'
for rep in "$@"; do
  name=$(basename "$rep" .ncu-rep)
  ncu -i "$rep" --page raw --csv 2>/dev/null | python3 -c "
import csv, re, sys
rows = list(csv.reader(sys.stdin))
hdr, units, data = rows[0], rows[1], rows[2:]
keep = [i for i, h in enumerate(hdr) if re.search(r'''$METRICS''', h)]
w = csv.writer(sys.stdout)
w.writerow([hdr[i] for i in keep]); w.writerow([units[i] for i in keep])
for r in data: w.writerow([r[i] for i in keep])
" > "profiles/$name.ncu-summary.csv"
  echo "profiles/$name.ncu-summary.csv: $(($(wc -l < profiles/$name.ncu-summary.csv) - 2)) kernel(s)"
done
